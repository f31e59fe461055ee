"""GPU: the float64 path (kernel 12) under the float64 error bounds of tests/f64_bounds.py, and its launch paths.

* Spectrogram rows at every window of ``f64_bounds.SWEEP`` (int16, float32, float64 input holding values float32
  cannot) under the spectrum bound; where nvcc is present, equal to the host build of the same transform within the
  margin of CUDA's hypot (2 ulp) against the host libm's (1 ulp): |a - b| <= 3 ulp of hypot, plus the two roundings of
  the division by K, 8 u relative.
* Chromagram rows, full and clipped frames (``parity.clipped_clips``), and feature rows 21-32 under the chroma bound;
  windows whose chroma tables the oracle refuses raise the same ValueError.
* Launch paths: both sides of the frame kernel's shared-memory cap (which instantiation ran, from a torch.profiler
  trace); more work items than the grid on the global-scratch path (2 x SMs CTAs) and on the shared-memory path (at most
  32 resident CTAs per SM x 4); ragged batches with poisoned padding, clips of no frames and refused clips, each clip
  equal to itself alone in bits.
* Beat on float64 rows whose peaks exist only in float64, bit for bit the host function.
Worst err / bound per window class is printed as JSON lines (DESIGN section 6)."""
import ctypes
import json
import re

import numpy as np
import pytest
import torch

from oracle import st_oracle as O
from pyaudioanalysis_b200 import batch as BT
from tests import f64_bounds as FB
from tests import host_exe
from tests import signals as SG
from tests.host_exe import bits, floats, hexes, run
from tests.kernels import GENERIC_SWEEP, ragged
from tests.parity import check_chromagram_bounds, chromagram_rows, clipped_clips, clipped_targets

pytestmark = pytest.mark.gpu

F64 = torch.float64
RT, AT = 1e-9, 1e-11
DTYPES = (np.int16, np.float32, np.float64)
CHROMA_CONFIGS = [(16000, 800, 300), (16000, 801, 333), (44100, 882, 441), (44100, 2205, 1000), (16000, 997, 400),
                  (44100, FB.SMEM_LAST, 2000), (44100, FB.BIG_FIRST, 2000)]
POISON = 0x7ff4dead0000beef
WORST = {}


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def note(key, r):
    WORST[key] = max(WORST.get(key, 0.0), r)


def window_class(w):
    if w >= FB.BIG_FIRST:
        return "global scratch"
    return "prime" if FB.radices(w) == [w] and w > 7 else ("w <= 33" if w <= 33 else "shared memory")


def spectrogram_frames(x, w, s):
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    starts = list(range(w, len(y) - w + 1, s))
    return np.stack([y[p:p + w] for p in starts]) if starts else np.zeros((0, w))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "f64_host.cu", "-O2")


@pytest.mark.parametrize("w", FB.SWEEP)
def test_spectrogram_rows_within_bound(w):
    fs = 44100 if w in (882, 2205, 44100, FB.SMEM_LAST, FB.BIG_FIRST) else 16000
    for dtype in DTYPES:
        x = FB.kind_clip(w, dtype)
        if dtype == np.float64:
            assert (x.astype(np.float32).astype(np.float64) != x).mean() > 0.9
        sp = BT.spectrogram_batch(dev(x), fs, w, w, dtype=F64)[0].cpu().numpy()
        fr = spectrogram_frames(x, w, w)
        assert len(fr) == len(FB.KINDS) and sp.shape[0] == len(fr) + 1
        assert not sp[len(fr):].any(), "rows the reference never fills are zero"
        r = FB.check_spectrum(sp[:len(fr)], fr, "spectrogram f64, w=%d, %s" % (w, np.dtype(dtype).name))
        note("spectrogram / " + window_class(w), r)
    print(json.dumps({"w": w, "worst": WORST}))


@pytest.mark.parametrize("w", [2, 9, 20, 21, 33, 882, 997, 2205, FB.SMEM_LAST, FB.BIG_FIRST, 20011, 44100])
def test_spectrogram_rows_equal_the_host_transform(harness, w):
    """The device runs the arithmetic the CPU tests verified: its rows equal the host build's hypot(re, im) / K within
    the two hypot implementations' documented errors."""
    x = FB.kind_clip(w, np.int16)
    sp = BT.spectrogram_batch(dev(x), 16000, w, w, dtype=F64)[0].cpu().numpy()
    fr = spectrogram_frames(x, w, w)
    out = run(harness, "".join("spec %d %s\n" % (w, hexes(f)) for f in fr))
    host = np.stack([floats(line[1:]) for line in out])
    err = np.abs(sp[:len(fr)] - host)
    assert (err <= 8 * FB.U64 * np.abs(host) + 1e-300).all(), (w, float((err / np.maximum(np.abs(host), 1e-300)).max()))


def _chroma_ok(fs, w):
    try:
        O.chroma_operator(fs, w // 2)
        return True
    except ValueError:
        return False


@pytest.mark.parametrize("fs,w,s", CHROMA_CONFIGS, ids=["%d-%d-%d" % c for c in CHROMA_CONFIGS])
def test_chromagram_rows_within_bound(fs, w, s):
    seen = set()
    for n_last in clipped_targets(w, s):
        clips = clipped_clips(fs, w, s, n_last)
        for dtype in (np.int16, np.float32):
            names = [k for k, v in clips.items() if v.dtype == dtype]
            xs = [clips[k] for k in names]
            d, lens = ragged(xs, dtype)
            out = BT.chromagram_batch(d, fs, w, s, lengths=lens, dtype=F64).cpu().numpy()
            for i, x in enumerate(xs):
                cb = FB.chromagram_bounds(x, fs, w, s)
                R = cb.ref.shape[0]
                assert not out[i, R:].any()
                worst, unb = check_chromagram_bounds(out[i, :R], cb, "f64 chromagram %d/%d/%d, last frame %d: %s"
                                                     % (fs, w, s, n_last, names[i]))
                assert not unb, unb
                for k, v in worst.items():
                    note("chromagram %s / %s" % (k, window_class(w)), v)
                    seen.add(k)
    assert {"full", "clipped"} <= seen
    # feature rows 21 .. 32 of full frames: the same fold over the same spectrum
    for dtype in DTYPES:
        x = FB.kind_clip(w, dtype)
        F = BT.feature_extraction_batch(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy()
        worst, unb = check_chromagram_bounds(F[21:33].T, FB.feature_chroma_bounds(x, fs, w, s),
                                             "f64 feature chroma rows %d/%d/%d %s" % (fs, w, s, np.dtype(dtype).name))
        assert not unb
        note("feature chroma / " + window_class(w), worst["full"])
    print(json.dumps({"config": [fs, w, s], "worst": WORST}))


@pytest.mark.parametrize("w", [c[1] for c in GENERIC_SWEEP if c[1] <= 33])
def test_refusals_follow_the_oracle(w):
    """Windows whose chroma tables the oracle refuses: chromagram and features raise its ValueError; the spectrogram
    still runs.  A clip too short for one row is refused as the oracle refuses it."""
    fs = 16000
    x = FB.kind_clip(w, np.int16)
    if not _chroma_ok(fs, w):
        with pytest.raises(ValueError):
            O.chromagram(x, fs, w, w)
        with pytest.raises(ValueError):
            BT.chromagram_batch(dev(x), fs, w, w, dtype=F64)
        with pytest.raises(ValueError):
            BT.feature_extraction_batch(dev(x), fs, w, w, dtype=F64)
    BT.spectrogram_batch(dev(x), fs, w, w, dtype=F64)
    short = x[:w - 1]
    with pytest.raises(ValueError):
        O.feature_extraction(short, fs, w, w)
    with pytest.raises(ValueError):
        BT.feature_extraction_batch(dev(short), fs, w, w, dtype=F64)


# ---------------------------------------------------------------------------------------------------------------------
# launch paths
def _frames_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {m.group(2) for e in prof.events() for m in [re.search(r"f64_frames_kernel<(\d+), (true|false)>", e.name)] if m}


@pytest.mark.parametrize("w,big", [(FB.SMEM_LAST, "false"), (FB.BIG_FIRST, "true")])
def test_both_sides_of_the_shared_memory_cap(w, big):
    fs, s = 44100, 2000
    x = O.synth_clip(w, 6 * w + 3 * s, fs)
    runs = {"features": lambda: BT.feature_extraction_batch(dev(x), fs, w, s, dtype=F64),
            "spectrogram": lambda: BT.spectrogram_batch(dev(x), fs, w, s, dtype=F64),
            "chromagram": lambda: BT.chromagram_batch(dev(x), fs, w, s, dtype=F64)}
    for name, fn in runs.items():
        assert _frames_kernels(fn) == {big}, (name, w)
    F = BT.feature_extraction_batch(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy()
    ref, _ = O.feature_extraction_loop(x, fs, w, s, tables_per_frame=False)
    np.testing.assert_allclose(F, ref, rtol=RT, atol=AT)


def _alone_in_bits(batch_out, clips, call, counts, what):
    """Clip i's first counts[i] rows (features: columns) of a batch equal the clip alone, in bits."""
    for i, x in enumerate(clips):
        if counts[i]:
            got = batch_out[i][:, :counts[i]] if what == "features" else batch_out[i][:counts[i]]
            np.testing.assert_array_equal(bits(got), bits(call(dev(x))[0].cpu().numpy()), err_msg="%s clip %d" % (what, i))


def _three_modes(xs, fs, w, s, oracle_clips=()):
    L = dev(np.array([x.size for x in xs], np.int64))
    d = dev(np.stack(xs))
    F = BT.feature_extraction_batch(d, fs, w, s, lengths=L, dtype=F64).cpu().numpy()
    _alone_in_bits(F, xs, lambda c: BT.feature_extraction_batch(c, fs, w, s, dtype=F64),
                   [O.frame_count(x.size, w, s) for x in xs], "features")
    sp = BT.spectrogram_batch(d, fs, w, s, lengths=L, dtype=F64)
    counts = BT.row_counts(L, w, s, 0).cpu().tolist()
    for i, x in enumerate(xs):
        alone = BT.spectrogram_batch(dev(x), fs, w, s, dtype=F64)[0]
        assert torch.equal(sp[i, :counts[i]].view(torch.int64), alone.view(torch.int64)), "spectrogram clip %d" % i
    del sp
    ch = BT.chromagram_batch(d, fs, w, s, lengths=L, dtype=F64).cpu().numpy()
    _alone_in_bits(ch, xs, lambda c: BT.chromagram_batch(c, fs, w, s, dtype=F64),
                   BT.row_counts(L, w, s, 1).cpu().tolist(), "chromagram")
    for i in oracle_clips:
        x = xs[i]
        ref, _ = O.feature_extraction_loop(x, fs, w, s, tables_per_frame=False)
        bad = SG.noise_defined_frames(x, w, s)
        ok = ~bad & ~np.concatenate([[False], bad[:-1]])
        np.testing.assert_allclose(F[i][:, ok], ref[:, ok], rtol=RT, atol=AT, err_msg="features clip %d" % i)
        np.testing.assert_allclose(BT.spectrogram_batch(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy(),
                                   O.spectrogram(x, fs, w, s)[0], rtol=RT, atol=AT, err_msg="spectrogram clip %d" % i)
        np.testing.assert_allclose(ch[i], O.chromagram(x, fs, w, s)[0], rtol=RT, atol=AT, err_msg="chromagram clip %d" % i)


def test_global_scratch_grid_stride():
    """12 three-minute clips at 44 100 / 44 100 / 22 050: more work items than the 2 x SMs CTAs of the global-scratch
    path, so every CTA reuses its scratch for several items, and segments start inside a clip (the flux's previous
    frame at t0 - 1)."""
    fs, w, s = 44100, 44100, 22050
    n = 180 * fs
    items = 12 * -(-O.frame_count(n, w, s) // 16)
    assert items > 2 * torch.cuda.get_device_properties(0).multi_processor_count
    xs = [O.synth_clip(300 + i, n, fs) for i in range(12)]
    assert _frames_kernels(lambda: BT.spectrogram_batch(dev(xs[0]), fs, w, s, dtype=F64)) == {"true"}
    _three_modes(xs, fs, w, s, oracle_clips=(0, 7))


def test_shared_memory_grid_stride():
    """96 clips of 30 s at 400 / 160: more work items than SMs x 32 resident CTAs x 4, the shared-memory grid's most."""
    fs, w, s = 16000, 400, 160
    n = 30 * fs
    items = 96 * -(-O.frame_count(n, w, s) // 16)
    assert items > torch.cuda.get_device_properties(0).multi_processor_count * 32 * 4
    xs = [O.synth_clip(500 + i, n, fs) for i in range(96)]
    _three_modes(xs, fs, w, s, oracle_clips=(3,))


def _refused_length(w, s):
    for n in range(2 * w, 6 * w):
        if chromagram_rows(n, w, s)[3] and chromagram_rows(n, w, s)[0] > 0:
            return n
    return None


RAGGED = [(44100, 441, 220), (44100, 882, 441), (16000, 801, 333), (8000, 257, 100), (16000, 16000, 8000)]


@pytest.mark.parametrize("fs,w,s", RAGGED, ids=["%d-%d-%d" % c for c in RAGGED])
def test_ragged_batches_poisoned(fs, w, s):
    """Frame counts = 0, 1, 15, 16, 17 (mod 16), clips of no frames and chromagram-refused clips, one ragged batch per
    mode into poisoned output: each clip's rows equal the clip alone in bits, everything past them keeps the poison."""
    from pyaudioanalysis_b200._lib import check, get_plan, lib
    lens = [w + (T - 1) * s + extra for T, extra in ((15, 0), (16, s // 2), (17, 1), (32, s - 1), (33, 0), (48, 3))]
    lens += [0, w - 1]
    r = _refused_length(w, s)
    if r:
        lens.append(r)
    rng = np.random.default_rng(w)
    xs = [np.round(rng.normal(0, 3000, n)).astype(np.int16) for n in lens]
    d, L = ragged(xs, np.int16)
    B, N = d.shape
    T = O.frame_count(N, w, s)
    out = torch.full((B, 68, T), 0, dtype=torch.int64, device="cuda").fill_(POISON).view(F64)
    F = BT.feature_extraction_batch(d, fs, w, s, lengths=L, out=out, dtype=F64).cpu().numpy()
    for i, x in enumerate(xs):
        Tb = O.frame_count(x.size, w, s)
        if Tb:
            np.testing.assert_array_equal(bits(F[i, :, :Tb]), bits(BT.feature_extraction_batch(dev(x), fs, w, s, dtype=F64)[0]
                                                                   .cpu().numpy()), err_msg="features clip %d" % i)
        assert (F[i, :, Tb:].view(np.int64) == POISON).all(), "features clip %d: padding written" % i
    norm = BT.clip_stats_f64(d, L)
    pl = get_plan(fs, w, s)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    seen = set()
    for which, fn, width, rows_of, entry in ((0, BT.spectrogram_batch, w // 2, lib().b200aa_spectrogram_rows,
                                              lib().b200aa_spectrogram_ragged_f64),
                                             (1, BT.chromagram_batch, 12, lib().b200aa_chromagram_rows,
                                              lib().b200aa_chromagram_ragged_f64)):
        R = rows_of(N, w, s)
        raw = torch.full((B, R, width), 0, dtype=torch.int64, device="cuda").fill_(POISON)
        check(entry(pl.handle, ctypes.c_void_p(d.data_ptr()), 0, B, N, d.stride(0), ctypes.c_void_p(L.data_ptr()),
                       ctypes.c_void_p(norm.data_ptr()), ctypes.c_void_p(raw.data_ptr()), stream))
        got = raw.cpu().numpy()
        counts = BT.row_counts(L, w, s, which).cpu().tolist()
        for i, x in enumerate(xs):
            try:
                alone = fn(dev(x), fs, w, s, dtype=F64)[0].cpu().numpy()
            except ValueError:
                alone = None
                seen.add("refused")
            assert counts[i] == (0 if alone is None else alone.shape[0]), (which, i)
            if alone is not None:
                assert (got[i, :counts[i]] == bits(alone)).all(), "mode %d clip %d differs from alone" % (which, i)
            assert (got[i, counts[i]:] == POISON).all(), "mode %d clip %d: padding written" % (which, i)
    assert "refused" in seen
    assert {O.frame_count(n, w, s) % 16 for n in lens} >= {0, 1, 15}


# ---------------------------------------------------------------------------------------------------------------------
# beat on float64 rows
def _host_beat(st, frames, window):
    import warnings
    from pyaudioanalysis_b200.MidTermFeatures import beat_extraction
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return np.array([beat_extraction(st[b, :, :frames[b]], window) for b in range(st.shape[0])])


def _walk_rows(B, T, seed):
    """Random walks of scale 1e-9 around 1.0: every peak is below float32 resolution (1.0 +- 6e-8 rounds to 1.0)."""
    rng = np.random.default_rng(seed)
    return 1.0 + 1e-9 * np.cumsum(rng.standard_normal((B, 34, T)), axis=2)


@pytest.mark.parametrize("T", [40, 1024, 1025, 4097])
def test_beat_on_float64_only_peaks(T):
    st = _walk_rows(5, T, T)
    st[2, 3, T // 2] = np.nan                               # a NaN row
    st[3, :, :] = np.nan
    frames = [T, T - 1, T // 2, T, 1]
    fr = dev(np.array(frames, np.int64))
    f32 = st.astype(np.float32).astype(np.float64)
    for window in (0.05, 0.025, 0.1, 0.8, 1.5, 0.0005):
        got = BT.beat_extraction_batch(dev(st), window, n_frames=fr, dtype=F64).cpu().numpy()
        host = _host_beat(st, frames, window)
        np.testing.assert_array_equal(bits(got), bits(host), err_msg="window %g" % window)
        if window < 0.5:            # a histogram of more than two bins: the walks' peaks decide it
            h32 = _host_beat(f32, frames, window)
            assert not np.array_equal(bits(host[[0, 1]]), bits(h32[[0, 1]])), "float32 rows give the same beat (%g)" % window

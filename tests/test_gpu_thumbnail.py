"""GPU: kernel 10 (b200aa_music_thumbnail) and the drop-in music_thumbnailing / self_similarity_matrix, bit for bit the
reference's scipy and NumPy steps: the stubbed-feature goldens and the planted-repeat track, tile edges, the NaN box rule,
ragged batches against one-track calls, batches over several scratch slices, strided and column-major inputs, and
concurrent streams and threads."""
import threading

import numpy as np
import pytest
import scipy.signal
import torch
from scipy.spatial import distance

from tests.host_exe import bits
from tests.thumb_cases import STUB_CASES, golden, planted_track
from pyaudioanalysis_b200 import ShortTermFeatures, audioSegmentation as A
from pyaudioanalysis_b200.batch import music_thumbnailing_batch
from pyaudioanalysis_b200.consumers import self_similarity_batch, thumbnail_batch

pytestmark = pytest.mark.gpu


def scipy_sim(X):
    with np.errstate(all="ignore"):
        return 1.0 - distance.squareform(distance.pdist(X, "cosine"))


def reference_steps(S, m, gap, limit_1=0, limit_2=1):
    """audioSegmentation.py:1145-1177 on a similarity matrix (the masking loop written as one array assignment)."""
    C = scipy.signal.convolve2d(S, np.eye(m, m), "valid")
    min_sm = np.min(C)
    i, j = np.indices(C.shape)
    C[(np.abs(i - j) < gap) | (i > j)] = min_sm
    C[0:int(limit_1 * C.shape[0]), :] = min_sm
    C[:, 0:int(limit_1 * C.shape[0])] = min_sm
    C[int(limit_2 * C.shape[0])::, :] = min_sm
    C[:, int(limit_2 * C.shape[0])::] = min_sm
    rows, cols = np.unravel_index(C.argmax(), C.shape)
    i1, i2, j1, j2 = rows, rows, cols, cols
    while i2 - i1 < m:
        if i1 <= 0 or j1 <= 0 or i2 >= C.shape[0] - 2 or j2 >= C.shape[1] - 2:
            break
        if C[i1 - 1, j1 - 1] > C[i2 + 1, j2 + 1]:
            i1, j1 = i1 - 1, j1 - 1
        else:
            i2, j2 = i2 + 1, j2 + 1
    return (i1, i2, j1, j2), C


def tbits(t):
    return bits(t.cpu().numpy())


def gpu_thumb(X, m, gap, limit_1=0, limit_2=1):
    idx, C = thumbnail_batch(torch.from_numpy(np.ascontiguousarray(X)).cuda(), [X.shape[0]], m, gap, limit_1, limit_2)
    return tuple(int(v) for v in idx[0]), C[0].cpu().numpy()


# ------------------------------------------------------------------ goldens of the unmodified reference
@pytest.mark.parametrize("name", list(STUB_CASES))
def test_stub_goldens(name, monkeypatch):
    """music_thumbnailing on the stubbed features: the four times (NumPy float64) and the masked matrix in bits, or the
    reference's exception; self_similarity_matrix's S in bits where stored."""
    g = golden()
    st = g[name + "_st"]
    monkeypatch.setattr(ShortTermFeatures, "feature_extraction", lambda *a, **k: (st.copy(), []))
    _, _, step, thumb, l1, l2, _ = STUB_CASES[name]
    err = str(g[name + "_error"])
    if err:
        with pytest.raises(ValueError):
            A.music_thumbnailing(np.zeros(16000, np.int16), 16000, 1.0, step, thumb, l1, l2)
    else:
        res = A.music_thumbnailing(np.zeros(16000, np.int16), 16000, 1.0, step, thumb, l1, l2)
        assert all(type(t) is np.float64 for t in res[:4])
        assert np.array_equal(bits(np.array(res[:4])), bits(g[name + "_times"]))
        assert isinstance(res[4], np.ndarray) and np.array_equal(bits(res[4]), bits(g[name + "_C"]))
    if name + "_S" in g.files:
        assert np.array_equal(bits(A.self_similarity_matrix(st)), bits(g[name + "_S"]))


@pytest.mark.parametrize("name,channels", [("planted", 1), ("planted_stereo", 2)])
def test_planted_repeat_end_to_end(name, channels):
    """With the drop-in's own features, the planted repeat gives the reference's exact times, mono and stereo."""
    res = A.music_thumbnailing(planted_track(channels=channels), 16000)
    assert np.array_equal(np.array(res[:4]), golden()["e2e_%s_times" % name])


def test_track_without_frames_raises():
    assert str(golden()["e2e_no_frames_error"]) == "ValueError"
    with pytest.raises(ValueError):
        A.music_thumbnailing(np.zeros(8000, np.int16), 16000)


# ------------------------------------------------------------------ tile edges and the NaN box rule
@pytest.mark.parametrize("F", [1, 2, 3, 67, 68, 69, 137])
def test_similarity_tile_edges(F):
    rng = np.random.default_rng(F)
    Ts = (1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 191, 193)
    X = [A.standardise(rng.normal(size=(F, T)) * 3 + rng.normal(size=(F, 1))) for T in Ts]
    got = self_similarity_batch(torch.from_numpy(np.concatenate(X)).cuda(), Ts)
    for T, x, S in zip(Ts, X, got):
        assert np.array_equal(tbits(S), bits(scipy_sim(x))), (F, T)


@pytest.mark.parametrize("T,F,m", [(31, 68, 1), (32, 3, 1), (33, 68, 2), (63, 1, 20), (64, 69, 20), (65, 137, 20),
                                   (95, 68, 64), (96, 2, 65), (150, 67, 33), (129, 68, 97)])
def test_filter_tile_edges(T, F, m):
    """R = T - m + 1 around multiples of the 32-wide filter tile and the 64-wide similarity tile."""
    rng = np.random.default_rng(T + F + m)
    X = A.standardise(rng.normal(size=(F, T)) + np.cos(np.arange(T) / 4.0))
    for gap, limits in ((10.0, (0, 1)), (0.5, (0.1, 0.95)), (3.0, (0.8, 0.2))):
        idx, C = gpu_thumb(X, m, gap, *limits)
        ridx, rC = reference_steps(scipy_sim(X), m, gap, *limits)
        assert idx == tuple(int(v) for v in ridx), (T, F, m, gap)
        assert np.array_equal(bits(C), bits(rC)), (T, F, m, gap)


@pytest.mark.parametrize("where", ["nan_feature", "zero_row", "overflow", "subnormal"])
def test_nan_box_rule(where):
    rng = np.random.default_rng(len(where))
    X = rng.normal(size=(140, 9))
    if where == "nan_feature":
        X[77, 4] = np.nan
    elif where == "zero_row":
        X[100] = 0.0
    elif where == "overflow":
        X[30:32] *= 1e300
    else:
        X[50] *= 1e-310
    for m in (1, 8, 40):
        idx, C = gpu_thumb(X, m, 5.0)
        ridx, rC = reference_steps(scipy_sim(X), m, 5.0)
        assert idx == tuple(int(v) for v in ridx), (where, m)
        assert np.array_equal(bits(C), bits(rC)), (where, m)


# ------------------------------------------------------------------ batches, slices, layouts
def _tracks(rng, Ts, F=68):
    return [A.standardise(rng.normal(size=(F, T)) + np.sin(np.arange(T) / rng.uniform(2, 9))) for T in Ts]


def _alone(X, m, gap, l1=0, l2=1):
    idx, C = thumbnail_batch(torch.from_numpy(X).cuda(), [X.shape[0]], m, gap, l1, l2)
    return idx[0], C[0]


def test_ragged_batch_equals_single_calls_with_poisoned_padding():
    """A ragged batch (a track shorter than the filter among them) read from rows whose padding columns are NaN."""
    rng = np.random.default_rng(5)
    Ts = [40, 300, 7, 129, 64, 21, 500]
    X = _tracks(rng, Ts)
    big = torch.full((sum(Ts), 75), float("nan"), dtype=torch.float64, device="cuda")
    big[:, :68] = torch.from_numpy(np.concatenate(X)).cuda()
    idx, C = thumbnail_batch(big[:, :68], Ts, 20, 10.0, 0.1, 0.9)
    for b, x in enumerate(X):
        i1, c1 = _alone(x, 20, 10.0, 0.1, 0.9)
        assert np.array_equal(idx[b], i1), b
        assert torch.equal(C[b].view(torch.int64), c1.view(torch.int64)), b


def test_column_major_input():
    rng = np.random.default_rng(6)
    x = _tracks(rng, [90])[0]
    cm = torch.from_numpy(np.asfortranarray(x)).cuda()
    assert cm.stride(1) != 1
    idx, C = thumbnail_batch(cm, [90], 12, 4.0)
    i1, c1 = _alone(x, 12, 4.0)
    assert np.array_equal(idx[0], i1) and torch.equal(C[0], c1)


def test_batch_over_several_scratch_slices_and_a_track_past_the_cap():
    """Tracks of 3 000 frames (four of them need two 256 MiB slices) and one of 6 000 frames (S alone is 288 MB, a slice
    of its own), against each track run alone."""
    rng = np.random.default_rng(7)
    Ts = [3000, 3000, 2999, 3001, 6000, 50]
    X = _tracks(rng, Ts, F=17)
    idx, C = thumbnail_batch(torch.from_numpy(np.concatenate(X)).cuda(), Ts, 20, 10.0)
    for b, x in enumerate(X):
        i1, c1 = _alone(x, 20, 10.0)
        assert np.array_equal(idx[b], i1), b
        assert torch.equal(C[b].view(torch.int64), c1.view(torch.int64)), b
    ridx, rC = reference_steps(scipy_sim(X[-1]), 20, 10.0)
    assert tuple(idx[-1]) == tuple(int(v) for v in ridx) and np.array_equal(bits(C[-1].cpu().numpy()), bits(rC))


def test_music_thumbnailing_batch_equals_one_track_calls():
    x = planted_track(seconds=60)
    clips = [x, x[:16000 * 25 + 3000], x[16000 * 8:16000 * 50], x[:16000 * 3]]
    N = max(len(c) for c in clips)
    sig = torch.zeros((len(clips), N), dtype=torch.int16)
    for b, c in enumerate(clips):
        sig[b, :len(c)] = torch.from_numpy(c)
        sig[b, len(c):] = 12345                                      # padding the lengths exclude
    lengths = torch.tensor([len(c) for c in clips], dtype=torch.int64).cuda()
    times, C = music_thumbnailing_batch(sig.cuda(), 16000, lengths=lengths)
    for b, c in enumerate(clips):
        res = A.music_thumbnailing(c, 16000)
        assert np.array_equal(bits(times[b]), bits(np.array(res[:4]))), b
        assert np.array_equal(tbits(C[b]), bits(res[4])), b


def test_streams_and_threads_share_the_entry():
    rng = np.random.default_rng(8)
    jobs = [_tracks(rng, [int(T)]) [0] for T in rng.integers(100, 700, size=8)]
    want = [_alone(x, 20, 10.0) for x in jobs]
    torch.cuda.synchronize()
    got = [None] * len(jobs)

    def work(k):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            X = torch.from_numpy(jobs[k]).cuda()
            idx, C = thumbnail_batch(X, [X.shape[0]], 20, 10.0)
            s.synchronize()
            got[k] = (idx[0], C[0])

    threads = [threading.Thread(target=work, args=(k,)) for k in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    for (i0, c0), (i1, c1) in zip(want, got):
        assert np.array_equal(i0, i1) and torch.equal(c0.view(torch.int64), c1.view(torch.int64))

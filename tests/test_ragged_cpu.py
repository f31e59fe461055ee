"""CPU: the chunk planner of the directory wrappers (MidTermFeatures._plan_chunks) and the argument checks of the ragged
pooling entry points, which return before touching a device."""
import ctypes

import numpy as np
import pytest

from pyaudioanalysis_b200.MidTermFeatures import _Clip, _plan_chunks, _MAX_CHUNK_BYTES, _MAX_PADDING

I16, F32 = 0, 1


def clips_of(spec):
    return [_Clip("f%d.wav" % i, fs, n, None, code) for i, (fs, n, code) in enumerate(spec)]


def folder(seed, n=400):
    rng = np.random.default_rng(seed)
    fs = rng.choice([8000, 16000, 44100], size=n)
    code = rng.choice([I16, F32], size=n, p=[0.8, 0.2])
    lens = rng.integers(1, 20 * 44100, size=n)
    lens[:20] = 160000                       # ties
    lens[20:30] = 160000 + np.arange(10)     # neighbours one sample apart
    return clips_of(zip(fs.tolist(), lens.tolist(), code.tolist()))


def check_plan(clips, chunks, max_bytes=_MAX_CHUNK_BYTES, max_padding=_MAX_PADDING):
    flat = [i for c in chunks for i in c]
    assert sorted(flat) == list(range(len(clips))), "every clip exactly once"
    for c in chunks:
        assert c, "no empty chunk"
        assert len({(clips[i].fs, clips[i].code) for i in c}) == 1, "one (rate, format) per chunk"
        ns = [clips[i].n for i in c]
        assert ns == sorted(ns, reverse=True), "longest first"
        item = 2 if clips[c[0]].code == I16 else 4
        if len(c) > 1:
            assert len(c) * ns[0] * item <= max_bytes, "staging cap"
            assert len(c) * ns[0] - sum(ns) <= max_padding * sum(ns), "padding bound"


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_planner_invariants(seed):
    clips = folder(seed)
    chunks = _plan_chunks(clips)
    check_plan(clips, chunks)
    assert chunks == _plan_chunks(clips), "deterministic"
    assert len(chunks) < len(clips) // 4, "clips of different lengths share chunks"


def test_planner_small_caps():
    clips = folder(3)
    for max_bytes, max_padding in ((1 << 20, 0.25), (4 << 20, 0.0), (1 << 30, 0.01), (1 << 30, 10.0)):
        chunks = _plan_chunks(clips, max_bytes=max_bytes, max_padding=max_padding)
        check_plan(clips, chunks, max_bytes, max_padding)


def test_planner_equal_lengths_one_chunk():
    clips = clips_of([(16000, 160000, I16)] * 1000)
    assert _plan_chunks(clips) == [list(range(1000))]
    chunks = _plan_chunks(clips, max_bytes=160000 * 2 * 300)        # room for 300 clips per chunk
    assert [len(c) for c in chunks] == [300, 300, 300, 100]


def test_planner_oversize_clip_alone():
    big = _MAX_CHUNK_BYTES // 2 + 1            # int16 samples: one clip is just over 1 GiB
    clips = clips_of([(16000, 1000, I16), (16000, big, I16), (16000, 999, I16), (16000, big // 2, F32),
                      (16000, big // 2 - 5, F32)])
    chunks = _plan_chunks(clips)
    check_plan(clips, chunks)
    assert [1] in chunks, "a clip larger than the cap is a chunk of its own"
    assert [0, 2] in chunks
    assert [3] in chunks and [4] in chunks, "two float32 clips of 512 MiB each exceed the cap together"


@pytest.fixture(scope="module")
def lib():
    from pyaudioanalysis_b200.build import build
    build()
    from pyaudioanalysis_b200 import _lib
    return _lib.lib()


def test_ragged_entry_points_reject_bad_arguments(lib):
    INVALID = -1
    p = ctypes.c_void_p(256)                   # never dereferenced: every call below fails its argument check first
    n = None
    # b200aa_frame_counts(d_len, n_clips, window, step, step_ratio, d_frames, d_windows, stream)
    assert lib.b200aa_frame_counts(n, 4, 800, 400, 1, p, p, n) == INVALID
    assert lib.b200aa_frame_counts(p, 4, 800, 400, 1, n, p, n) == INVALID
    assert lib.b200aa_frame_counts(p, 4, 800, 400, 0, p, p, n) == INVALID
    assert lib.b200aa_frame_counts(p, 4, 0, 400, 1, p, p, n) == INVALID
    assert lib.b200aa_frame_counts(p, 4, 800, 0, 1, p, n, n) == INVALID
    assert lib.b200aa_frame_counts(p, -1, 800, 400, 1, p, n, n) == INVALID
    # b200aa_mid_pool_ragged(d_st, n_clips, n_feats, t_stride, d_frames, ratio, step_ratio, d_mid, stream)
    assert lib.b200aa_mid_pool_ragged(n, 2, 68, 100, p, 39, 40, p, n) == INVALID
    assert lib.b200aa_mid_pool_ragged(p, 2, 68, 100, n, 39, 40, p, n) == INVALID
    assert lib.b200aa_mid_pool_ragged(p, 2, 68, 100, p, 39, 40, n, n) == INVALID
    assert lib.b200aa_mid_pool_ragged(p, 2, 68, 100, p, 39, 0, p, n) == INVALID
    assert lib.b200aa_mid_pool_ragged(p, 2, 68, 100, p, 39, -3, p, n) == INVALID
    assert lib.b200aa_mid_pool_ragged(p, 2, 0, 100, p, 39, 40, p, n) == INVALID
    assert lib.b200aa_mid_pool_ragged(p, 2, 68, -1, p, 39, 40, p, n) == INVALID
    # b200aa_long_term_mean_ragged(d_mid, n_clips, n_rows, m_stride, d_windows, d_out, stream)
    assert lib.b200aa_long_term_mean_ragged(n, 2, 136, 10, p, p, n) == INVALID
    assert lib.b200aa_long_term_mean_ragged(p, 2, 136, 10, n, p, n) == INVALID
    assert lib.b200aa_long_term_mean_ragged(p, 2, 136, 10, p, n, n) == INVALID
    assert lib.b200aa_long_term_mean_ragged(p, 2, 0, 10, p, p, n) == INVALID
    assert lib.b200aa_long_term_mean_ragged(p, 2, 136, -1, p, p, n) == INVALID


def test_ragged_python_api_refuses_cpu_tensors():
    import torch
    import pyaudioanalysis_b200 as pkg
    with pytest.raises(TypeError):
        pkg.frame_counts(torch.zeros(3, dtype=torch.int64), 800, 400)
    with pytest.raises(TypeError):
        pkg.mid_pool_batch(torch.zeros(2, 68, 10), 3, 2, n_frames=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(TypeError):
        pkg.long_term_mean_batch(torch.zeros(2, 136, 10), n_windows=torch.zeros(2, dtype=torch.int64))

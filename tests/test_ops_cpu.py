"""CPU: the ``torch.ops.b200aa`` operators (pyaudioanalysis_b200/ops.py) are registered with a fake implementation on a
machine without a GPU, and the shapes those give are the library's counts.

* Every operator exists after ``import pyaudioanalysis_b200`` and runs on fake CUDA tensors under ``FakeTensorMode``.
* The Python counts equal ``b200aa_num_frames``, ``b200aa_spectrogram_rows``, ``b200aa_chromagram_rows`` and
  ``b200aa_mid_windows`` for every clip length 0 .. 3 w + 2 s of each (window, step) below, step > window and windows
  that clip chromagram frames included, and their refusals equal csrc/rows.cuh's (run on the host by tests/rows_host.cu).
* The fake implementations give those shapes, float windows and steps truncated as ``int()`` truncates them, and raise
  ValueError wherever the eager call refuses the shape.
* They also trace with symbolic sizes (``make_fx(tracing_mode="symbolic")``).
"""
import pytest

from tests import host_exe

# (window, step): hop below, at and above the window; odd windows; chromagram frames clipped short of w / 2 and not
CONFIGS = [(800, 400), (800, 333), (800, 800), (800, 1200), (882, 441), (400, 160), (2, 1), (5, 3), (7, 10), (16, 5),
           (31, 4), (30, 30)]


@pytest.fixture(scope="module")
def env():
    import torch
    import pyaudioanalysis_b200 as pkg
    from pyaudioanalysis_b200 import _lib
    return torch, pkg, _lib.lib()


@pytest.fixture(scope="module")
def rows_ref(tmp_path_factory):
    """(w, s) -> {n: (spec_R, spec_refused, chroma_R, chroma_refused)} from csrc/rows.cuh on the host."""
    exe = host_exe.build(tmp_path_factory, "rows_host.cu", "-O1")
    out = host_exe.run(exe, "".join("%d %d %d\n" % (w, s, 3 * w + 2 * s) for w, s in CONFIGS))
    ref, i = {}, 0
    for w, s in CONFIGS:
        i += 1                                  # the max_clipped line
        table = {}
        for _ in range(3 * w + 2 * s + 1):
            t = [int(v) for v in out[i]]
            table[t[0]] = (t[1], bool(t[4]), t[5], bool(t[8]))
            i += 1
        ref[(w, s)] = table
    return ref


def test_every_op_registered_with_fake(env):
    torch, pkg, _ = env
    from torch._subclasses.fake_tensor import FakeTensorMode
    assert set(pkg.ops.OPS) == {"clip_stats", "feature_extraction", "spectrogram", "chromagram", "frame_counts",
                                "row_counts", "mid_pool", "mid_feature_extraction", "long_term_mean", "beat_extraction"}
    ops = torch.ops.b200aa
    with FakeTensorMode():
        x = torch.empty(3, 16000, dtype=torch.int16, device="cuda")
        lens = torch.empty(3, dtype=torch.int64, device="cuda")
        st = torch.empty(3, 68, 39, dtype=torch.float32, device="cuda")
        shapes = {
            "clip_stats": ops.clip_stats(x).shape,
            "clip_stats f64": ops.clip_stats(x, lens, torch.float64).shape,
            "feature_extraction": ops.feature_extraction(x, 16000, 800, 400, lengths=lens).shape,
            "spectrogram": ops.spectrogram(x, 16000, 800, 400).shape,
            "chromagram": ops.chromagram(x, 16000, 800, 400, dtype=torch.float64).shape,
            "frame_counts": tuple(t.shape for t in ops.frame_counts(lens, 800, 400, 10)),
            "row_counts": ops.row_counts(lens, 800, 400, 1).shape,
            "mid_pool": ops.mid_pool(st, 19, 10).shape,
            "mid_feature_extraction": tuple(t.shape for t in ops.mid_feature_extraction(x, 16000, 8000, 4000, 800, 400)),
            "long_term_mean": ops.long_term_mean(st, lens).shape,
            "beat_extraction": ops.beat_extraction(st, 0.025, lens).shape,
        }
        assert ops.clip_stats(x).dtype == torch.uint8 and ops.beat_extraction(st, 0.025).dtype == torch.float64
        assert ops.feature_extraction(x, 16000, 800, 400, dtype=torch.float64).dtype == torch.float64
    assert shapes == {
        "clip_stats": (3, 32), "clip_stats f64": (3, 16), "feature_extraction": (3, 68, 39), "spectrogram": (3, 39, 400),
        "chromagram": (3, 38, 12), "frame_counts": ((3,), (3,)), "row_counts": (3,), "mid_pool": (3, 136, 4),
        "mid_feature_extraction": ((3, 136, 4), (3, 68, 39)), "long_term_mean": (3, 68), "beat_extraction": (3, 2)}


@pytest.mark.parametrize("w,s", CONFIGS)
def test_counts_equal_library(env, rows_ref, w, s):
    _, pkg, L = env
    O = pkg.ops
    for n in range(3 * w + 2 * s + 1):
        spec_R, spec_ref, chroma_R, chroma_ref = rows_ref[(w, s)][n]
        assert O.num_frames(n, w, s) == L.b200aa_num_frames(n, w, s), n
        assert O.spectrogram_rows(n, w, s) == (L.b200aa_spectrogram_rows(n, w, s), spec_ref) == (spec_R, spec_ref), n
        assert O.chromagram_rows(n, w, s) == (L.b200aa_chromagram_rows(n, w, s), chroma_ref) == (chroma_R, chroma_ref), n
        for stepr in (1, 2, 3, 10):
            T = L.b200aa_num_frames(n, w, s)
            assert O.mid_windows(T, stepr) == L.b200aa_mid_windows(T, stepr), (n, stepr)
    assert O.mid_windows(5, 0) == L.b200aa_mid_windows(5, 0) == 0


def _fake_shape(torch, fn):
    """The shape a fake call gives, or "refused" when it raises ValueError."""
    from torch._subclasses.fake_tensor import FakeTensorMode
    with FakeTensorMode():
        try:
            out = fn()
        except ValueError:
            return "refused"
    return tuple(tuple(t.shape) for t in out) if isinstance(out, tuple) else tuple(out.shape)


# float (window, step) arguments and the ints they truncate to
FLOAT_ARGS = [((800.9, 400.2), (800, 400)), ((7.5, 10.99), (7, 10)), ((16.0, 5.7), (16, 5)), ((30.3, 30.9), (30, 30))]


@pytest.mark.parametrize("fw,fs_,w,s", [(a, b, c, d) for (a, b), (c, d) in FLOAT_ARGS])
def test_fake_shapes_and_refusals(env, rows_ref, fw, fs_, w, s):
    torch, _, L = env
    ops = torch.ops.b200aa
    B = 2
    for n in range(3 * w + 2 * s + 1):
        spec_R, spec_ref, chroma_R, chroma_ref = rows_ref[(w, s)][n]

        def clips(n=n):
            return torch.empty(B, n, dtype=torch.int16, device="cuda")

        def lens():
            return torch.empty(B, dtype=torch.int64, device="cuda")

        T = L.b200aa_num_frames(n, w, s)
        assert _fake_shape(torch, lambda: ops.feature_extraction(clips(), 16000, fw, fs_)) == \
            ((B, 68, T) if T > 0 else "refused"), n
        assert _fake_shape(torch, lambda: ops.feature_extraction(clips(), 16000, fw, fs_, False, lens())) == \
            ((B, 34, T) if T > 0 else "refused"), n
        want = (B, spec_R, w // 2) if not spec_ref else "refused"
        assert _fake_shape(torch, lambda: ops.spectrogram(clips(), 16000, fw, fs_)) == want, n
        assert _fake_shape(torch, lambda: ops.spectrogram(clips(), 16000, fw, fs_, lens())) == want, n
        assert _fake_shape(torch, lambda: ops.chromagram(clips(), 16000, fw, fs_)) == \
            ((B, chroma_R, 12) if not chroma_ref else "refused"), n
        assert _fake_shape(torch, lambda: ops.chromagram(clips(), 16000, fw, fs_, lens())) == \
            ((B, chroma_R, 12) if chroma_R > 0 else "refused"), n
        # mid-term windows of 3 and 10 steps (ratio and step ratio from the raw arguments, as mid_feature_extraction)
        for mid_w, mid_s in ((3 * fs_, 3 * fs_), (10 * fs_ + fw, 10 * fs_)):
            stepr = int(round(mid_s / fs_))
            want = ((B, 136, L.b200aa_mid_windows(T, stepr)), (B, 68, T)) if T > 0 else "refused"
            assert _fake_shape(torch, lambda: ops.mid_feature_extraction(clips(), 16000, mid_w, mid_s, fw, fs_)) == want


def test_fake_refusals_of_arguments(env):
    torch, _, _ = env
    ops = torch.ops.b200aa

    def refused(fn):
        return _fake_shape(torch, fn) == "refused"

    x = lambda n=16000: torch.empty(2, n, dtype=torch.int16, device="cuda")     # noqa: E731
    st = lambda T=39, F=68, dt=torch.float32: torch.empty(2, F, T, dtype=dt, device="cuda")     # noqa: E731
    lens = lambda: torch.empty(2, dtype=torch.int64, device="cuda")     # noqa: E731
    assert refused(lambda: ops.mid_feature_extraction(x(), 16000, 8000, 150, 800, 400))         # step ratio round(0.375) < 1
    assert refused(lambda: ops.mid_pool(st(), 19, 0))
    assert refused(lambda: ops.mid_pool(st(T=0), 19, 10))                                       # no frames to pool
    assert not refused(lambda: ops.mid_pool(st(T=0), 19, 10, lens()))                           # ragged: none is allowed
    assert _fake_shape(torch, lambda: ops.mid_pool(st(T=0), 19, 10, lens())) == (2, 136, 0)
    assert refused(lambda: ops.long_term_mean(st(T=0)))
    assert _fake_shape(torch, lambda: ops.long_term_mean(st(T=0), lens())) == (2, 68)
    assert refused(lambda: ops.beat_extraction(st(F=18), 0.025))
    assert refused(lambda: ops.beat_extraction(st(), 5.0))                                      # round(0.4) = 0 bins
    assert refused(lambda: ops.feature_extraction(x(), 16000, 1, 1))                            # window < 2: no plan
    assert refused(lambda: ops.feature_extraction(x(), 16000, 800, 0.5))                        # step truncates to 0
    assert refused(lambda: ops.frame_counts(lens(), 800, 400, 0))
    assert refused(lambda: ops.row_counts(lens(), 800, 400, 2))
    with pytest.raises(TypeError):
        _fake_shape(torch, lambda: ops.feature_extraction(x(), 16000, 800, 400, dtype=torch.float16))


def test_fakes_trace_with_symbolic_sizes(env):
    torch, _, _ = env
    from torch.fx.experimental.proxy_tensor import make_fx

    def f(x, lens):
        mid, st = torch.ops.b200aa.mid_feature_extraction(x, 16000, 8000, 4000, 800, 400, lens)
        frames, windows = torch.ops.b200aa.frame_counts(lens, 800, 400, 10)
        return (torch.ops.b200aa.long_term_mean(mid, windows), torch.ops.b200aa.beat_extraction(st, 0.025, frames),
                torch.ops.b200aa.spectrogram(x, 16000, 800, 333), torch.ops.b200aa.chromagram(x, 16000, 800, 333, lens))

    x = torch.empty(3, 16123, dtype=torch.int16, device="meta")
    lens = torch.empty(3, dtype=torch.int64, device="meta")
    gm = make_fx(f, tracing_mode="symbolic")(x, lens)
    outs = [n for n in gm.graph.nodes if n.op == "call_function"]
    assert any("mid_feature_extraction" in str(n.target) for n in outs)
    got = [tuple(t.shape) for t in gm(torch.empty(3, 20000, dtype=torch.int16, device="meta"), lens)]
    assert got == [(3, 136), (3, 2), (3, (20000 - 800) // 333 + 1, 400), (3, (20000 - 333 - 800) // 333 + 1, 12)]

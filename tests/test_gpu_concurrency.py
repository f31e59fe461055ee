"""GPU: every entry point under concurrent streams and host threads that share one plan gives, bit for bit, what the same
call gives alone on the default stream.

A cached plan (``get_plan``) is handed to every caller of the process, whatever its thread or stream, and the C ABI's
device entry points are asynchronous on the caller's stream.  What that sharing reaches: the plan's ring of 64 work
slots (csrc/slots.h: a slot in flight is never handed to a second launch, a reused slot's stream waits on its last
user), the stream-ordered scratch of the large-window generic kernel, the large-window clipped-chromagram kernel, beat
extraction and PCM decode, the three streams of the chunked host pipeline and the lock around the host-buffer
workspaces.  No kernel waits for another CTA, so a launch whose CTAs are not all resident at once (another stream's
kernel holds SMs) still finishes.

* Baseline: every job alone on the default stream, synchronised; its outputs, its ``b200aa_launch_count()`` delta and,
  from the ``B200AA_DEBUG`` launcher lines, how many slot-taking launches (pair, solo, CTA kernel) it made.
* Phase A: one thread, 4 streams, the jobs round-robin over them, no host synchronisation until the end; the slot-taking
  jobs repeat until each of their plans gets at least 3 x 64 slots, so every ring comes round at least three times.
* Phase B: 6 threads, each on its own stream, released together, interleaving the device jobs (together about as many
  runs as phase A, so the rings again come round at least three times) with the host-buffer entry points
  (``ShortTermFeatures``, ``MidTermFeatures.mid_feature_extraction``, ``HostPipeline.run`` single-stream and chunked
  over three streams) on the same plans.
* Every output equals its baseline as integer bits, the zero columns / rows past each clip's own counts included.  The
  launch count of each phase is the sum of its jobs' baseline counts.  One output of every kernel kind is also held to
  its float64 bound (``parity.feature_bounds``, ``check_spectrogram_rows``, ``chromagram_bounds``).
* Bit-equal results are promised for int16 input.  Float32 clip statistics add doubles with atomics in no fixed order:
  the float32 feature jobs take the baseline's records as ``norm=``, and the concurrent float32 ``clip_stats`` are held
  to the exact-arithmetic check of ``parity.check_f32_clip``.

Inputs are made before a phase on the default stream, which every stream waits on; outputs passed as ``out=`` are
allocated there too, the others by the entry point on the job's stream.  Every tensor is held until the final
synchronisation.  A fixed number of jobs, no retries, no timing assertion.
"""
import json
import threading

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import wavgen
from tests.kernels import CTA, GENERIC, PAIR, SOLO, ragged
from tests.parity import (check_f32_clip, check_feature_bounds, check_rows, check_spectrogram_rows, chromagram_bounds,
                          feature_bounds)

pytestmark = pytest.mark.gpu

STREAMS, THREADS, RING = 4, 6, 64
SLOT_LAUNCHERS = ("[b200aa] pair kernel", "[b200aa] solo kernel", "[b200aa] fast kernel")
MID = (8000, 4000)                      # mid-term window / step in samples at 16 kHz


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


def launches():
    from pyaudioanalysis_b200._lib import lib
    return lib().b200aa_launch_count()


def bits(o):
    import torch
    a = np.ascontiguousarray(o.cpu().numpy() if isinstance(o, torch.Tensor) else o)
    return a.view({1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}[a.dtype.itemsize])


class Job:
    """One call of an entry point: ``run(out)`` queues it on the current stream (a host-buffer entry point runs it to the
    end) and returns its outputs; ``alloc()`` makes the ``out=`` argument beforehand on the default stream.  ``plan``
    names the plan whose ring it takes slots from; ``check``, when given, replaces the bit comparison."""

    def __init__(self, name, run, plan=None, alloc=None, check=None, reps=8, threads=True):
        self.name, self.run, self.plan, self.alloc, self.check = name, run, plan, alloc or (lambda: None), check
        self.reps, self.threads = reps, threads
        self.base = self.launches = self.slots = None


def clips16(seed, lengths, fs):
    return [O.synth_clip(seed + i, n, fs) for i, n in enumerate(lengths)]


def wav_clips(P, tmp_path, flavours, tag):
    from pyaudioanalysis_b200.MidTermFeatures import _open_clip
    out = []
    for k, (name, ch) in enumerate(flavours):
        p = str(tmp_path / ("%s%d_%s_%d.wav" % (tag, k, name, ch)))
        wavgen.write(p, 16000, wavgen.signal(name, ch, 7000 + 1531 * k, 90 + k), name)
        out.append(_open_clip(p))
    assert all(c.data is None for c in out)
    return out


def make_jobs(P, tmp_path):
    """(device jobs, host jobs, bound checks on the baseline's outputs); the jobs hold their inputs."""
    import torch
    from pyaudioanalysis_b200 import audioio, consumers
    from pyaudioanalysis_b200._lib import Plan, get_plan
    from pyaudioanalysis_b200.hostpipe import HostPipeline
    ST, M = P.ShortTermFeatures, P.MidTermFeatures
    plans = {"pair": get_plan(16000, 800, 400), "solo": get_plan(44100, 882, 441),
             "CTA": Plan(16000, 800, 400).prefer_kernel(CTA), "generic": Plan(16000, 800, 400),
             "generic 20000": Plan(16000, 20000, 10000)}
    plans["generic"].force_generic(True)
    plans["generic 20000"].force_generic(True)
    for name, kind in (("pair", PAIR), ("solo", SOLO), ("CTA", CTA), ("generic", GENERIC), ("generic 20000", GENERIC)):
        assert plans[name].kernel_kind() == kind, name

    # inputs: ragged int16 batches whose clips end in partial hops (clipped chromagram frames), float32 copies
    x16 = clips16(10, [16000, 12345, 9999, 7001], 16000)
    d16, l16 = ragged(x16, np.int16)
    f16 = [(x.astype(np.float32) * np.float32(0.37) + np.float32(11.5)) for x in x16]
    df16, lf16 = ragged(f16, np.float32)
    x44 = clips16(20, [44100, 30011, 22050], 44100)
    d44, l44 = ragged(x44, np.int16)
    x20k = clips16(30, [64001, 50000, 43210], 16000)
    d20k, l20k = ragged(x20k, np.int16)
    big = torch.from_numpy(np.stack(clips16(40, [160000] * 4, 16000) * 64)).cuda()          # 256 clips of 10 s
    ratio, stepr = O.mid_ratios(MID[0], MID[1], 800, 400)
    fnorm = P.clip_stats(df16, lf16)
    st_in = P.feature_extraction_batch(d16, 16000, 800, 400, lengths=l16)
    frames, windows = P.frame_counts(l16, 800, 400, step_ratio=stepr)
    mid_in = P.mid_pool_batch(st_in, ratio, stepr, n_frames=frames)
    rng = np.random.default_rng(5)
    mean = rng.normal(0, 1, 136).astype(np.float32)
    std = rng.uniform(0.5, 2, 136).astype(np.float32)
    wav16 = wav_clips(P, tmp_path, [("s16", 1), ("u8", 1), ("s16", 1)], "i")
    wavf = wav_clips(P, tmp_path, [("s24", 2), ("f32", 1), ("s16", 2), ("f64", 2), ("s32", 1)], "f")
    T16 = O.frame_count(d16.shape[1], 800, 400)

    def zeros(*shape):
        return lambda: torch.zeros(shape, dtype=torch.float32, device="cuda")

    def feats(d, lens, fs, w, s, plan, deltas=True, norm=None):
        return lambda out: (P.feature_extraction_batch(d, fs, w, s, deltas=deltas, out=out, lengths=lens, norm=norm,
                                                       plan=None if plan is None else plans[plan]),)

    def f32_stats(out):
        rec = out[0].view(torch.float32).cpu().numpy()
        for i, x in enumerate(f16):
            check_f32_clip(rec[i], x, "float32 clip_stats, clip %d" % i)

    dev = [
        Job("pair features", feats(d16, l16, 16000, 800, 400, None), "pair", zeros(4, 68, T16), reps=RING),
        Job("pair features, no deltas", feats(d16, l16, 16000, 800, 400, None, deltas=False), "pair", zeros(4, 34, T16),
            reps=RING),
        Job("pair features, float32", feats(df16, lf16, 16000, 800, 400, None, norm=fnorm), "pair", zeros(4, 68, T16),
            reps=RING),
        Job("pair features, 256 x 10 s", feats(big, None, 16000, 800, 400, None), "pair", reps=4, threads=False),
        Job("solo features", feats(d44, l44, 44100, 882, 441, None), "solo", reps=RING),
        Job("solo spectrogram", lambda out: (P.spectrogram_batch(d44, 44100, 882, 441, lengths=l44),), "solo", reps=RING),
        Job("solo chromagram", lambda out: (P.chromagram_batch(d44, 44100, 882, 441, lengths=l44),), "solo", reps=RING),
        Job("CTA features", feats(d16, l16, 16000, 800, 400, "CTA"), "CTA", reps=RING),
        Job("CTA spectrogram", lambda out: (P.spectrogram_batch(d16, 16000, 800, 400, plan=plans["CTA"], lengths=l16),),
            "CTA", reps=RING),
        Job("CTA chromagram", lambda out: (P.chromagram_batch(d16, 16000, 800, 400, plan=plans["CTA"], lengths=l16),),
            "CTA", reps=RING),
        Job("generic features", feats(d16, l16, 16000, 800, 400, "generic"), "generic"),
        Job("generic chromagram", lambda out: (P.chromagram_batch(d16, 16000, 800, 400, plan=plans["generic"], lengths=l16),),
            "generic"),
        Job("generic features, window 20000", feats(d20k, l20k, 16000, 20000, 10000, "generic 20000"), "generic 20000",
            reps=2),
        Job("generic chromagram, window 20000",
            lambda out: (P.chromagram_batch(d20k, 16000, 20000, 10000, plan=plans["generic 20000"], lengths=l20k),),
            "generic 20000", reps=2),
        Job("clip_stats int16", lambda out: (P.clip_stats(d16, l16, out=out),),
            alloc=lambda: torch.zeros((4, 32), dtype=torch.uint8, device="cuda")),
        Job("clip_stats float32", lambda out: (P.clip_stats(df16, lf16, out=out),), check=f32_stats,
            alloc=lambda: torch.zeros((4, 32), dtype=torch.uint8, device="cuda")),
        Job("frame_counts", lambda out: P.frame_counts(l16, 800, 400, step_ratio=stepr)),
        Job("row_counts", lambda out: (P.row_counts(l16, 800, 400, 0), P.row_counts(l44, 882, 441, 1))),
        Job("mid_pool_batch", lambda out: (P.mid_pool_batch(st_in, ratio, stepr, n_frames=frames),)),
        Job("long_term_mean_batch", lambda out: (P.long_term_mean_batch(mid_in, n_windows=windows),)),
        Job("beat_extraction_batch", lambda out: (P.beat_extraction_batch(st_in, 400 / 16000, n_frames=frames),)),
        Job("normalize_windows_batch", lambda out: (consumers.normalize_windows_batch(mid_in, mean, std),)),
        Job("PCM decode, int16", lambda out: audioio.stage(wav16), reps=2),
        Job("PCM decode, float32", lambda out: audioio.stage(wavf), reps=2),
    ]

    # host-buffer entry points on the same cached plans
    hx = x16[0]
    hx44 = x44[1]
    single = HostPipeline(16000, 800, 400, 16000, 8, bind_numa=False)
    single.h_in[:] = np.stack(clips16(50, [16000] * 8, 16000))
    n_long = 960000                     # 60 s clips: the chunked path cuts 32 MB chunks of 17 clips; 36 clips = 3 chunks
    chunked = HostPipeline(16000, 800, 400, n_long, 36, bind_numa=False)
    chunked.h_in[:] = np.random.default_rng(6).integers(-20000, 20000, (36, n_long), dtype=np.int16)
    host = [
        Job("ShortTermFeatures.feature_extraction", lambda out: (ST.feature_extraction(hx, 16000, 800, 400)[0],), "pair"),
        Job("ShortTermFeatures.spectrogram", lambda out: (ST.spectrogram(hx44, 44100, 882, 441)[0],), "solo"),
        Job("ShortTermFeatures.chromagram", lambda out: (ST.chromagram(hx44, 44100, 882, 441)[0],), "solo"),
        Job("MidTermFeatures.mid_feature_extraction", lambda out: M.mid_feature_extraction(hx, 16000, *MID, 800, 400)[:2],
            "pair"),
        Job("HostPipeline.run, one stream", lambda out: (single.run(out=out),), "pair",
            alloc=lambda: np.zeros((8, 68, single.T), np.float32)),
        Job("HostPipeline.run, three streams", lambda out: (chunked.run(out=out),), "pair",
            alloc=lambda: np.zeros((36, 68, chunked.T), np.float32)),
    ]

    def bound_checks(base):
        """One output per kernel kind against its float64 bound."""
        accs = {}
        for job, x in (("pair features", x16), ("CTA features", x16), ("generic features", x16), ("solo features", x44)):
            fs, w, s = (44100, 882, 441) if job.startswith("solo") else (16000, 800, 400)
            out = base[job][0]
            for i, xi in enumerate(x):
                fb = feature_bounds(xi, fs, w, s, deltas=True)
                T = fb.ref.shape[1]
                assert not out[i, :, T:].any(), "%s: clip %d: columns past its frames" % (job, i)
                check_feature_bounds(out[i, :, :T], fb, "%s, clip %d" % (job, i))
        for job, x, (fs, w, s) in (("solo chromagram", x44, (44100, 882, 441)), ("CTA chromagram", x16, (16000, 800, 400)),
                                   ("generic chromagram", x16, (16000, 800, 400))):
            check_rows(base[job][0], [chromagram_bounds(xi, fs, w, s) for xi in x], ["%s, clip %d" % (job, i) for i in range(len(x))],
                       accs, (job, "int16"))
        sp = base["solo spectrogram"][0]
        for i, xi in enumerate(x44):
            R = int((xi.size - 882) / 441) + 1
            assert not sp[i, R:].any(), "solo spectrogram, clip %d: rows past its own" % i
            check_spectrogram_rows(sp[i, :R], xi, 882, 441, "solo spectrogram, clip %d" % i)
        return accs

    return dev, host, bound_checks


def expect_equal(job, out, what):
    if job.check is not None:
        job.check(out)
        return
    assert len(out) == len(job.base), (what, job.name)
    for k, (o, b) in enumerate(zip(out, job.base)):
        g = bits(o)
        assert g.shape == b.shape and np.array_equal(g, b), "%s: %s, output %d differs from the job alone (%d of %d elements)" % (
            what, job.name, k, int((g != b).sum()) if g.shape == b.shape else -1, b.size)


def test_concurrent_equals_serial(P, tmp_path, monkeypatch, capfd):
    import torch
    monkeypatch.setattr(P.ShortTermFeatures, "PRINT_SPECTROGRAM_SHAPE", False)
    dev, host, bound_checks = make_jobs(P, tmp_path)
    torch.cuda.synchronize()

    # ---- baseline: each job alone on the default stream
    monkeypatch.setenv("B200AA_DEBUG", "1")
    base_out = {}
    for job in dev + host:
        capfd.readouterr()
        n0 = launches()
        out = job.run(job.alloc())
        torch.cuda.synchronize()
        job.launches = launches() - n0
        job.slots = sum(ln.startswith(SLOT_LAUNCHERS) for ln in capfd.readouterr().err.splitlines())
        assert (job.slots > 0) == (job.plan in ("pair", "solo", "CTA")), (job.name, job.slots)
        assert job.launches >= 1, job.name
        base_out[job.name] = [o.cpu().numpy() if isinstance(o, torch.Tensor) else np.array(o) for o in out]
        if job.check is not None:
            job.check(out)
        job.base = [bits(o) for o in out]
    monkeypatch.delenv("B200AA_DEBUG")
    accs = bound_checks(base_out)

    report = {"launches": {}, "slots": {}, "wraps": {}}

    def tally(phase, runs):
        slots = {}
        for job in runs:
            if job.slots:
                slots[job.plan] = slots.get(job.plan, 0) + job.slots
        report["slots"][phase] = slots
        report["wraps"][phase] = {k: v // RING for k, v in slots.items()}
        return sum(job.launches for job in runs), slots

    # ---- phase A: one thread, STREAMS streams, no host synchronisation until the end
    default = torch.cuda.current_stream()
    streams = [torch.cuda.Stream() for _ in range(STREAMS)]
    order = [job for r in range(max(j.reps for j in dev)) for job in dev if r < job.reps]
    prepared = [(job, job.alloc()) for job in order]
    for s in streams:
        s.wait_stream(default)
    n0 = launches()
    results = []
    for k, (job, o) in enumerate(prepared):
        with torch.cuda.stream(streams[k % STREAMS]):
            results.append((job, o, job.run(o)))
    torch.cuda.synchronize()
    got = launches() - n0
    want, slots = tally("A", order)
    report["launches"]["A"] = got
    assert got == want, "phase A: %d launches, the jobs alone make %d" % (got, want)
    for name in ("pair", "solo", "CTA"):
        assert slots.get(name, 0) >= 3 * RING, "phase A: plan %s took %d slots, fewer than three rings" % (name, slots.get(name, 0))
    for job, _, out in results:
        expect_equal(job, out, "phase A (%d streams, one thread)" % STREAMS)
    del results, prepared

    # ---- phase B: THREADS threads, each on its own stream, released together
    per_thread = [job for job in dev if job.threads for _ in range(-(-job.reps // THREADS))] + host
    barrier = threading.Barrier(THREADS, timeout=300)
    outs, errors = [None] * THREADS, []

    def worker(t):
        try:
            rng = np.random.default_rng(100 + t)
            mine = [per_thread[i] for i in rng.permutation(len(per_thread))]
            prep = [(job, job.alloc()) for job in mine]
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            barrier.wait()
            res = []
            with torch.cuda.stream(s):
                for job, o in prep:
                    res.append((job, o, job.run(o)))
            outs[t] = res
        except BaseException as e:           # noqa: BLE001 -- re-raised on the main thread
            errors.append(e)
            barrier.abort()

    n0 = launches()
    threads = [threading.Thread(target=worker, args=(t,)) for t in range(THREADS)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    torch.cuda.synchronize()
    if errors:
        raise errors[0]
    got = launches() - n0
    want, slots = tally("B", per_thread * THREADS)
    report["launches"]["B"] = got
    assert got == want, "phase B: %d launches, the jobs alone make %d" % (got, want)
    for name in ("pair", "solo", "CTA"):
        assert slots.get(name, 0) >= 3 * RING, "phase B: plan %s took %d slots, fewer than three rings" % (name, slots.get(name, 0))
    for t, res in enumerate(outs):
        for job, _, out in res:
            expect_equal(job, out, "phase B (thread %d of %d)" % (t, THREADS))
    worst = {"%s %s" % k: {n: round(v, 4) for n, v in acc["worst"].items()} for k, acc in accs.items()}
    with capfd.disabled():
        print(json.dumps(dict(report, chromagram_worst=worst)))


def test_kernel13_mixed_shapes_concurrent_equals_alone():
    """Kernel 13's batched entry points of different shapes on six threads, each on its own stream and with no lock, two
    calls of different shapes per build kernel: forest model selection (random forest at 11 features and 3 classes;
    extra trees at 512 features and 32 classes), forest regression model selection at 136 and at 11 features, and
    gradient boosting model selection at 40 features and 10 classes and at 512 features and 3 classes.  Each kernel's
    two callers need different amounts of dynamic shared memory; every launcher sets the kernel's limit to the one size
    of its largest accepted shape, so no thread's setting can undercut another's launch (a launcher that set its own
    size could fail the larger call, when the interleaving falls that way; tests/test_smem_budget_cpu.py checks the rule
    itself deterministically).
    Each thread makes its call three times; every result equals, in bits, the same call made alone beforehand.  Seeds
    are explicit, so no call touches NumPy's global state."""
    import torch
    from pyaudioanalysis_b200.consumers import (boosting_cross_validate, forest_cross_validate,
                                                forest_regression_cross_validate)

    def splits_of(r, n, P, n_train):
        out = []
        for _ in range(P):
            perm = r.permutation(n)
            out.append((perm[:n_train], perm[n_train:]))
        return out

    def forest_job(seed, n, F, C, kind, trees):
        r = np.random.RandomState(seed)
        y = (np.arange(n) % C).astype(np.float64)
        X = torch.from_numpy(r.randn(n, F) + 0.4 * (y[:, None] % 3 == np.arange(F) % 3)).cuda()
        sp = splits_of(r, n, len(trees), int(0.8 * n))
        seeds = [[int(s) for s in r.randint(0, 2 ** 31 - 1, T)] for T in trees]
        return lambda: forest_cross_validate(X, y, sp, seeds, trees, kind, n_classes=C)

    def regression_job(seed, n, F, trees):
        r = np.random.RandomState(seed)
        Xh = r.randn(n, F)
        X, y = torch.from_numpy(Xh).cuda(), Xh[:, 2] + 0.3 * r.randn(n)
        sp = splits_of(r, n, len(trees), int(0.8 * n))
        seeds = [[int(s) for s in r.randint(0, 2 ** 31 - 1, T)] for T in trees]
        return lambda: forest_regression_cross_validate(X, y, sp, seeds, trees)

    def boosting_job(seed, n, F, C, stages):
        r = np.random.RandomState(seed)
        y = r.permutation(np.arange(n) % C).astype(np.float64)
        X = torch.from_numpy(r.randn(n, F) + (y[:, None] == np.arange(F) % C)).cuda()
        sp = splits_of(r, n, len(stages), int(0.8 * n))
        K = [np.unique(y[tr]).size for tr, _ in sp]
        K = [1 if k == 2 else k for k in K]
        seeds = [r.randint(0, 2 ** 31 - 1, T * k).astype(np.uint32) for T, k in zip(stages, K)]
        return lambda: boosting_cross_validate(X, y, sp, seeds, stages, n_classes=C)

    jobs = [forest_job(81, 300, 11, 3, "randomforest", [6, 4]),
            forest_job(82, 320, 512, 32, "extratrees", [3, 2]),
            regression_job(83, 250, 136, [3, 2]),
            regression_job(85, 300, 11, [4, 3]),
            boosting_job(84, 300, 40, 10, [2, 3]),
            boosting_job(86, 240, 512, 3, [3, 2])]
    alone = []
    for job in jobs:
        out = job()
        torch.cuda.synchronize()
        alone.append([bits(o) for o in out])
    reps, results, errors = 3, [[None] * 3 for _ in jobs], []
    barrier = threading.Barrier(len(jobs))

    def worker(i):
        try:
            s = torch.cuda.Stream()
            barrier.wait()
            with torch.cuda.stream(s):
                for k in range(reps):
                    results[i][k] = jobs[i]()
            s.synchronize()
        except BaseException as e:           # noqa: BLE001 -- re-raised on the main thread
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=worker, args=(i,)) for i in range(len(jobs))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    torch.cuda.synchronize()
    if errors:
        raise errors[0]
    for i, (want, got) in enumerate(zip(alone, results)):
        for k, out in enumerate(got):
            for a, b in zip(want, out):
                assert np.array_equal(a, bits(b)), (i, k)

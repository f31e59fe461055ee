"""GPU: every chromagram entry of every row kernel kind, full-frame and clipped, within its per-entry bound
(``tests/parity.chromagram_bounds``, derivation in ``tests/test_chroma_bounds_cpu.py``).

* every row kernel kind ``tests.kernels.plans`` reaches (the pair kernel has no row mode) at ROW_CONFIGS and 800 / 200:
  the bank uncut as ragged int16 and float32 batches, the bank cut to its shortest clip through the equal-length entry
  point, and clips built to end in clipped frames (``clipped_clips``);
* the generic kernel's chromagram mode (``force_generic``) across ``tests.kernels.GENERIC_SWEEP``, on ``sweep_clips`` plus
  clips that end in a clipped frame; where the reference refuses the window (the chroma table at a tiny K) the call must
  raise the same error;
* the clipped-frame kernel directly: clipped lengths K, K + 1, a prime and w - 1 where reachable, at windows 800, 883,
  882 (44.1 kHz), both sides of its shared-memory / global-scratch boundary (8 900 / 8 901) and 16 000 / 8 000, on noise, DC
  20000 +- 3 LSB, a loud first sample, a tone whose other classes are ~1e-10 of the total, +-1 LSB dither, an exact
  integer-mean run (exact zeros) and float32 input at offset 11.5 and 1e-3 scale; in one ragged batch and through the
  equal-length path; and 800 / 100, whose (w - 1) / s = 7 candidate clipped frames per clip always include one shorter
  than K, so every such clip is refused.

Each test prints the worst err / bound per kernel, input type and row class as JSON lines.
"""
import json

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import GENERIC_SWEEP, KIND_NAMES, PAIR, ROW_CONFIGS, plans, ragged
from tests.parity import (check_rows, chromagram_bounds, chromagram_rows, clipped_clips, clipped_targets, ragged_bounds,
                          report)
from tests.signals import sweep_clips

pytestmark = pytest.mark.gpu

CONFIGS = ROW_CONFIGS + [(16000, 800, 200)]
CLIPPED_WINDOWS = [(16000, 800, 400), (16000, 800, 200), (16000, 883, 300), (44100, 882, 441), (16000, 8900, 4450),
                   (16000, 8901, 4450), (16000, 16000, 8000)]


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


@pytest.mark.parametrize("fs,w,s", CONFIGS, ids=["%d-%d-%d" % c for c in CONFIGS])
def test_rows_within_bound(P, fs, w, s):
    import torch
    ints, flts = SG.bank(fs, w, s), SG.float_bank(fs, w, s)
    clipped = {"%s_n%d" % (name, n): x for n in clipped_targets(w, s) for name, x in clipped_clips(fs, w, s, n).items()}
    cints = {k: v for k, v in clipped.items() if v.dtype == np.int16}
    cflts = {k: v for k, v in clipped.items() if v.dtype == np.float32}
    sets = [(bank, dtype, cls) for bank, dtype, cls in ((ints, np.int16, "int16"), (flts, np.float32, "float32"),
                                                        (cints, np.int16, "int16"), (cflts, np.float32, "float32"))]
    bounds = [[chromagram_bounds(x, fs, w, s) for x in bank.values()] for bank, _, _ in sets]
    cut = []
    for bank, dtype, cls in sets[:2]:
        n = min(x.size for x in bank.values())
        xs = [x[:n] for x in bank.values()]
        cut.append((xs, dtype, cls, [chromagram_bounds(x, fs, w, s) for x in xs]))
    accs = {}
    for kind, pl in plans(fs, w, s):
        if kind == PAIR:
            continue                      # the pair kernel has no row mode: the CTA kernel serves these rows
        name = KIND_NAMES[kind]
        for (bank, dtype, cls), cbs in zip(sets, bounds):
            tag = "%s rows, fs=%d w=%d s=%d, ragged" % (name, fs, w, s)
            ragged_bounds(P, pl, list(bank.values()), list(bank), dtype, fs, w, s, tag, accs, (name, cls), cbs)
        for (xs, dtype, cls, cbs), names in zip(cut, (list(ints), list(flts))):
            out = P.chromagram_batch(torch.from_numpy(np.stack(xs)).cuda(), fs, w, s, plan=pl).cpu().numpy()
            check_rows(out, cbs, ["%s rows, fs=%d w=%d s=%d, equal length: %s" % (name, fs, w, s, n) for n in names],
                       accs, (name, cls))
    report("%d-%d-%d" % (fs, w, s), accs)


@pytest.mark.parametrize("fs,w,G,path", GENERIC_SWEEP, ids=["w%d" % c[1] for c in GENERIC_SWEEP])
def test_generic_chromagram_within_bound(P, fs, w, G, path):
    import torch
    from pyaudioanalysis_b200._lib import Plan
    s, ints, flt = sweep_clips(w)
    try:
        O.chroma_operator(fs, w // 2)
        refused = None
    except ValueError as e:
        refused = type(e)
    if refused is not None:
        with pytest.raises(refused):
            pl = Plan(fs, w, s)
            pl.force_generic(True)
            d, lens = ragged(ints, np.int16)
            P.chromagram_batch(d, fs, w, s, plan=pl, lengths=lens)
        print(json.dumps(dict(config="generic w=%d" % w, refused=refused.__name__)))
        return
    pl = Plan(fs, w, s)
    pl.force_generic(True)
    targets = clipped_targets(w, s)
    extra = clipped_clips(fs, w, s, targets[-1]) if targets else {}
    clips = ints + [extra[k] for k in ("tone", "loud_first", "mean_run") if k in extra]
    names = ["int16 clip %d" % i for i in range(len(ints))] + [k for k in ("tone", "loud_first", "mean_run") if k in extra]
    accs = {}
    tag = "generic chromagram, w=%d s=%d (%s)" % (w, s, path)
    cbs = ragged_bounds(P, pl, clips, names, np.int16, fs, w, s, tag, accs, ("generic", "int16"))
    assert any((cb.cls == 1).any() for cb in cbs), tag + ": no clipped frame"
    fclips = [flt] + ([extra["small_f32"]] if extra else [])
    for x, nm in zip(fclips, ("float32 chirp", "small_f32")):
        out = P.chromagram_batch(torch.from_numpy(x).cuda()[None], fs, w, s, plan=pl).cpu().numpy()
        check_rows(out, [chromagram_bounds(x, fs, w, s)], ["%s: %s" % (tag, nm)], accs, ("generic", "float32"))
    report("generic w=%d G=%d" % (w, G), accs)


@pytest.mark.parametrize("fs,w,s", CLIPPED_WINDOWS, ids=["%d-%d-%d" % c for c in CLIPPED_WINDOWS])
def test_clipped_kernel_within_bound(P, fs, w, s):
    """The clipped-frame signals at every reachable target length, as one ragged batch per input type and again per length
    through the equal-length path (bit for bit the same rows for int16)."""
    import torch
    accs = {}
    by_len = {}
    for n in clipped_targets(w, s):
        for name, x in clipped_clips(fs, w, s, n).items():
            by_len.setdefault((x.size, x.dtype.name), []).append(("%s_n%d" % (name, n), x))
    cbs = {}
    for dtype, cls in ((np.int16, "int16"), (np.float32, "float32")):
        items = [it for (L, dt), its in by_len.items() if dt == np.dtype(dtype).name for it in its]
        names, clips = [k for k, _ in items], [x for _, x in items]
        cb = ragged_bounds(P, None, clips, names, dtype, fs, w, s, "clipped kernel, fs=%d w=%d s=%d, ragged" % (fs, w, s),
                           accs, ("clipped", cls))
        assert all((c.cls == 1).any() for c in cb)
        for k, c in zip(names, cb):
            cbs[k] = c
        d, lens = ragged(clips, dtype)
        rag = P.chromagram_batch(d, fs, w, s, lengths=lens)
        for (L, dt), its in by_len.items():
            if dt != np.dtype(dtype).name:
                continue
            out = P.chromagram_batch(torch.from_numpy(np.stack([x for _, x in its])).cuda(), fs, w, s)
            what = ["clipped kernel, fs=%d w=%d s=%d, equal length: %s" % (fs, w, s, k) for k, _ in its]
            check_rows(out.cpu().numpy(), [cbs[k] for k, _ in its], what, accs, ("clipped", cls + ", equal length"))
            if dtype == np.int16:
                for j, (k, _) in enumerate(its):
                    i = names.index(k)
                    assert torch.equal(out[j], rag[i, :out.shape[1]]), what[j] + ": differs from the ragged batch"
        for k, c in cbs.items():
            if k.startswith("mean_run"):
                assert not c.bound[-1].any(), k          # the integer-mean run: a zero bound, so exact zeros
    report("clipped %d-%d-%d" % (fs, w, s), accs)


def test_clipped_candidates_all_refused(P):
    """800 / 100: the loop's last frame has at most 2 s = 200 < K samples, so every clip with a row to fill is refused
    however many of its (w - 1) / s = 7 candidate clipped frames it has: no rows in a ragged batch, ValueError through the
    equal-length path.  A clip of w + s samples has one row that the loop never fills: exactly zero."""
    import torch
    fs, w, s = 16000, 800, 100
    rng = np.random.default_rng(11)
    lengths = [2 * w + 7 * s + d for d in (1, 50, 99)] + [5 * w + 33, w + s]
    clips = [np.round(rng.normal(0, 3000.0, n)).astype(np.int16) for n in lengths]
    rows = [chromagram_rows(n, w, s) for n in lengths]
    assert [r[3] for r in rows] == [True] * 4 + [False] and max(r[1] - r[2] for r in rows) == 7, rows
    accs = {}
    ragged_bounds(P, None, clips, ["%d samples" % n for n in lengths], np.int16, fs, w, s, "800 / 100", accs, ("default", "int16"))
    for x, r in zip(clips, rows):
        if r[3]:
            with pytest.raises(ValueError):
                P.chromagram_batch(torch.from_numpy(x).cuda()[None], fs, w, s)
    report("800-100", accs)

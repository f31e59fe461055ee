"""GPU: every short-term kernel across sample rates (tests.kernels.RATE_CONFIGS), where its tables take the layouts the
suite's 8 / 16 / 44.1 / 48 kHz configs never reach: empty mel filters (44.1 kHz and above at short windows), long lane
lists (up to 18 four-tap steps at 6 854 Hz, the lowest rate whose mel bank builds), the clamped group at that rate, chroma
lists of 9 and 10 taps, and hops longer than the window, where frames skip samples.  The layouts themselves are decoded
on the host by tests/test_rates_cpu.py.

For every kernel kind ``tests.kernels.plans`` reaches, on the adversarial bank plus ``odd_tail`` as ragged int16 and
float32 batches:

* the 68 feature rows, deltas on and off, within ``parity.feature_bounds``;
* the row kinds' chromagram within ``parity.chromagram_bounds`` and spectrogram rows within the spectrum bound
  (``parity.check_spectrogram_rows``);
* the kernel that ran is the one asked for: with ``B200AA_DEBUG`` set the pair, solo and CTA launchers print one line per
  launch and the generic kernel none.  A launcher that declines a shape falls through to the next kernel silently, and
  the values would still be right: this is what tells the two apart.  At 800 / 1600 the CTA kernel's staging is over its
  cap by design (tests/test_rates_cpu.CTA_FALLBACK) and the generic kernel runs: that is asserted too.

Entries with an unbounded bound are counted per reason and printed with the worst err / bound per kernel and input.

Reach of defects planted by hand in ``build_pair_blob`` (not committed), from the blobs they build on the host: an
empty filter that is not flushed, or the clamp moved one bin down (s2 = K - 5, the filter's last tap dropped), leaves
the pair blob bit-identical at every (fs, window) the rest of the GPU suite runs, so that suite cannot fail on them; the
configs here with empty filters / at 6 854 Hz change.  Moved one bin up (s2 = K - 3) the clamp reads one float past the
row against a zero weight: only the host decoder of tests/test_rates_cpu.py sees it.  Lane lists truncated at LQ = 8
and chroma lists truncated at CT = 8 already change the blob at 8 kHz / 600 (and, for CT, 16 kHz / 512, 1024,
44.1 kHz / 882, 48 kHz / 960), which the rest of the suite runs.  The planted defects were not run on the GPU.
"""
import json
import os

import numpy as np
import pytest

from tests import signals as SG
from tests.kernels import CTA, GENERIC, KIND_NAMES, PAIR, RATE_CONFIGS, SOLO, plans, ragged
from tests.parity import check_spectrogram_rows
from tests.test_gpu_chroma_bounds import ragged_bounds
from tests.test_gpu_feature_bounds import batch_bounds
from tests.test_gpu_spectra import odd_tail
from tests.test_rates_cpu import CTA_FALLBACK

pytestmark = pytest.mark.gpu

LAUNCHERS = {PAIR: "pair kernel", SOLO: "solo kernel", CTA: "fast kernel"}


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


@pytest.fixture
def debug(monkeypatch):
    monkeypatch.setenv("B200AA_DEBUG", "1")


def ran(capfd, expect, what):
    """The launcher lines printed since the last call name kernel `expect` (None: the generic kernel, which prints none)."""
    import torch
    torch.cuda.synchronize()
    err = capfd.readouterr().err
    lines = [ln for ln in err.splitlines() if ln.startswith("[b200aa]")]
    names = {name for name in LAUNCHERS.values() if any(ln.startswith("[b200aa] " + name) for ln in lines)}
    want = set() if expect is None else {expect}
    assert names == want, "%s: launched %s, expected %s" % (what, sorted(names) or "the generic kernel", expect or "the generic kernel")


def accumulate(accs, key, worst, unb):
    acc = accs.setdefault(key, {"worst": {}, "unbounded": {}})
    for k, v in worst.items():
        acc["worst"][k] = max(acc["worst"].get(k, 0.0), v)
    for k, v in unb.items():
        acc["unbounded"][k] = acc["unbounded"].get(k, 0) + v


@pytest.mark.parametrize("fs,w,s,kinds,layout", RATE_CONFIGS, ids=["%d-%d-%d" % c[:3] for c in RATE_CONFIGS])
def test_kernels_across_rates(P, debug, capfd, fs, w, s, kinds, layout):
    ints = dict(SG.bank(fs, w, s), odd_tail=odd_tail(fs, w, s))
    flts = dict(SG.float_bank(fs, w, s), odd_tail_f32=ints["odd_tail"].astype(np.float32) * np.float32(0.37) + np.float32(11.5))
    tag = "%d-%d-%d" % (fs, w, s)
    accs = {}
    seen = set()
    for kind, pl in plans(fs, w, s):
        seen.add(kind)
        name = KIND_NAMES[kind]
        expect = LAUNCHERS.get(kind)
        if kind == CTA and (w, s) in CTA_FALLBACK:
            expect = None
        for bank, dtype, cls in ((ints, np.int16, "int16"), (flts, np.float32, "float32")):
            what = ["%s kernel, fs=%d w=%d s=%d (%s): %s" % (name, fs, w, s, layout, n) for n in bank]
            acc = accs.setdefault(("features", name, cls), {"worst": {}, "unbounded": {}})
            capfd.readouterr()
            batch_bounds(P, pl, list(bank.values()), dtype, fs, w, s, what, acc)
            ran(capfd, expect, "%s features, %s %s" % (name, tag, cls))
            if kind == PAIR:
                continue                  # the pair kernel has no row mode
            rtag = "%s rows, fs=%d w=%d s=%d (%s), ragged" % (name, fs, w, s, layout)
            ragged_bounds(P, pl, list(bank.values()), list(bank), dtype, fs, w, s, rtag, accs, ("chromagram", name, cls))
            ran(capfd, expect, "%s chromagram, %s %s" % (name, tag, cls))
            d, lens = ragged(list(bank.values()), dtype)
            sp = P.spectrogram_batch(d, fs, w, s, plan=pl, lengths=lens).cpu().numpy()
            ran(capfd, expect, "%s spectrogram, %s %s" % (name, tag, cls))
            for i, (n, x) in enumerate(bank.items()):
                R = int((x.size - w) / s) + 1
                assert not sp[i, R:].any(), "%s: %s: rows past the clip's own" % (rtag, n)
                bins, dc = check_spectrogram_rows(sp[i, :R], x, w, s, "%s: %s spectrogram" % (rtag, n))
                accumulate(accs, ("spectrogram", name, cls), {"bins": bins, "dc": dc}, {})
    assert seen == kinds, (seen, kinds)
    assert GENERIC in seen
    for (what, kernel, cls), acc in accs.items():
        print(json.dumps(dict(config=tag, output=what, kernel=kernel, input=cls,
                              worst={k: round(v, 4) for k, v in acc["worst"].items()}, unbounded=acc["unbounded"])))

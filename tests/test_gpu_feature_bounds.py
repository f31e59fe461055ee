"""GPU: every feature entry of every kernel kind within its per-entry bound (``tests/parity.feature_bounds``, derivation
in ``tests/test_feature_bounds_cpu.py``), with no exception list and no rolloff flip allowance.

* every kernel kind ``tests.kernels.plans`` reaches at each adversarial feature config: the bank as one ragged int16
  batch and one ragged float32 batch, deltas on and off, plus ``odd_tail`` (an odd frame count whose last frame is loud in
  one half only);
* the generic kernel's feature mode (``force_generic``) across ``tests.kernels.GENERIC_SWEEP`` on the short clips of
  ``sweep_clips``; where the reference refuses the window (mel range or chroma tables at a tiny K) the kernel must raise
  the same error.

Entries whose bound is unbounded (a mel band whose interval reaches 0) are counted per reason and printed with the worst
err / bound of each row group.
"""
import json

import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import GENERIC_SWEEP, KIND_NAMES, plans, ragged
from tests.parity import check_feature_bounds, feature_bounds
from tests.test_gpu_adversarial import FEATURE_CONFIGS
from tests.test_gpu_spectra import odd_tail, sweep_clips

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


def note(acc, worst, unb):
    for k, v in worst.items():
        acc["worst"][k] = max(acc["worst"].get(k, 0.0), v)
    for k, v in unb.items():
        acc["unbounded"][k] = acc["unbounded"].get(k, 0) + v


def report(tag, accs):
    for key, acc in accs.items():
        print(json.dumps(dict(config=tag, kernel=key[0], input=key[1],
                              worst={k: round(v, 4) for k, v in acc["worst"].items()}, unbounded=acc["unbounded"])))


def batch_bounds(P, pl, clips, dtype, fs, w, s, what, acc):
    """clips as one ragged batch through plan pl, deltas on and off, every clip under its bound; rows past a clip's
    frame count stay zero."""
    d, lens = ragged(clips, dtype)
    fbs = [feature_bounds(x, fs, w, s, deltas=True) for x in clips]
    for deltas in (True, False):
        out = P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl, deltas=deltas).cpu().numpy()
        for i, fb in enumerate(fbs):
            T = fb.ref.shape[1]
            F = 68 if deltas else 34
            assert not out[i, :, T:].any(), what[i] + ": output past the clip's frames"
            if not deltas:
                fb = type(fb)(fb.ref[:34], fb.bound[:34], fb.roll, {k: v for k, v in fb.unbounded.items()
                                                                    if not k.startswith("delta")}, fb.K)
            note(acc, *check_feature_bounds(out[i, :F, :T], fb, what[i] + (", deltas" if deltas else ", no deltas")))


@pytest.mark.parametrize("fs,w,s,kinds", FEATURE_CONFIGS, ids=["%d-%d-%d" % c[:3] for c in FEATURE_CONFIGS])
def test_features_within_bound(P, fs, w, s, kinds):
    ints = dict(SG.bank(fs, w, s), odd_tail=odd_tail(fs, w, s))
    flts = dict(SG.float_bank(fs, w, s), odd_tail_f32=ints["odd_tail"].astype(np.float32) * np.float32(0.37) + np.float32(11.5))
    seen = set()
    accs = {}
    for kind, pl in plans(fs, w, s):
        seen.add(kind)
        for bank, dtype, cls in ((ints, np.int16, "int16"), (flts, np.float32, "float32")):
            acc = accs.setdefault((KIND_NAMES[kind], cls), {"worst": {}, "unbounded": {}})
            what = ["%s kernel, fs=%d w=%d s=%d: %s" % (KIND_NAMES[kind], fs, w, s, n) for n in bank]
            batch_bounds(P, pl, list(bank.values()), dtype, fs, w, s, what, acc)
    assert seen == kinds, (seen, kinds)
    report("%d-%d-%d" % (fs, w, s), accs)


@pytest.mark.parametrize("fs,w,G,path", GENERIC_SWEEP, ids=["w%d" % c[1] for c in GENERIC_SWEEP])
def test_generic_features_within_bound(P, fs, w, G, path):
    import torch
    from pyaudioanalysis_b200._lib import Plan
    s, ints, flt = sweep_clips(w)
    try:
        O.feature_extraction(ints[0], fs, w, s)
        refused = None
    except (IndexError, ValueError) as e:
        refused = type(e)
    if refused is not None:
        with pytest.raises(refused):
            pl = Plan(fs, w, s)
            pl.force_generic(True)
            d, lens = ragged(ints, np.int16)
            P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl)
        print(json.dumps(dict(config="generic w=%d" % w, refused=refused.__name__)))
        return
    pl = Plan(fs, w, s)
    pl.force_generic(True)
    acc = {"worst": {}, "unbounded": {}}
    batch_bounds(P, pl, ints, np.int16, fs, w, s, ["generic features, w=%d s=%d (%s): int16 clip %d" % (w, s, path, i)
                                                   for i in range(len(ints))], acc)
    fb = feature_bounds(flt, fs, w, s, deltas=True)
    out = P.feature_extraction_batch(torch.from_numpy(flt).cuda()[None], fs, w, s, plan=pl).cpu().numpy()
    note(acc, *check_feature_bounds(out[0], fb, "generic features, w=%d s=%d (%s): float32 chirp" % (w, s, path)))
    report("generic w=%d G=%d" % (w, G), {("generic", "sweep"): acc})

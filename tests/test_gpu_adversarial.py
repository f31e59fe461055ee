"""GPU: every short-term kernel against the float64 oracle on the adversarial signal bank (tests/signals.py).

For each (fs, window, hop) the whole bank runs as one ragged int16 batch through every kernel kind the plan can reach
(2 pair, 3 solo, 1 CTA, 0 generic), with deltas on and off; the float32 variants run through every kind too.  Every
clip is held to the standard feature tolerance (with the exceptions listed in tests/parity.EXCEPTIONS), its energy
row relative to its own level, and the zcr row of integer input to float32 rounding of the exact count.  int16 results
do not depend on the batch: a clip computed alone equals the same clip in the batch bit for bit, and so does a strided
view whose rows start at an odd sample offset (unaligned: no vector loads, no TMA), except through the CTA kernel,
where a row stride that is not a multiple of 8 samples selects a different staging variant: there the clip alone and
the view are held to the tolerance instead.
"""
import numpy as np
import pytest

from oracle import st_oracle as O
from tests import signals as SG
from tests.kernels import CTA, FEATURE_CONFIGS, KIND_NAMES, PAIR, ROW_CONFIGS, plans, ragged
from tests.parity import (check_close, check_energy_relative, check_features, check_spectrogram_rows, check_zcr_exact,
                          exception_bounds)

pytestmark = pytest.mark.gpu

ODD = 3                 # sample offset of the unaligned view


@pytest.fixture(scope="module")
def P():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    import pyaudioanalysis_b200 as pkg
    return pkg


def oracle_features(x, fs, w, s):
    """Oracle matrix (deltas on) with the noise-defined rows of constant frames set to their exact values."""
    xx = x.astype(np.float64) if x.dtype == np.float32 else x
    return SG.patch_noise_defined(O.feature_extraction(xx, fs, w, s)[0], x, w, s)[0]


def check_clip(got, ref, K, kind, name, what, integer):
    check_features(got, ref, K, what, allow=exception_bounds(name, kind))
    check_energy_relative(got, ref, what)
    if integer:
        check_zcr_exact(got, ref, what)


@pytest.mark.parametrize("fs,w,s,kinds", FEATURE_CONFIGS, ids=["%d-%d-%d" % c[:3] for c in FEATURE_CONFIGS])
def test_features_every_kernel(P, fs, w, s, kinds):
    import torch
    K = w // 2
    ints = SG.bank(fs, w, s)
    flts = SG.float_bank(fs, w, s)
    names, clips = list(ints), list(ints.values())
    fnames, fclips = list(flts), list(flts.values())
    refs = [oracle_features(x, fs, w, s) for x in clips]
    frefs = [oracle_features(x, fs, w, s) for x in fclips]
    T = [r.shape[1] for r in refs]
    d, lens = ragged(clips, np.int16)
    dodd, _ = ragged(clips, np.int16, offset=ODD)
    assert d.data_ptr() % 16 == 0 and d.stride(0) % 8 == 0 and dodd.data_ptr() % 16 != 0 and dodd.stride(0) % 8 != 0
    df, flens = ragged(fclips, np.float32)
    seen = set()
    for kind, pl in plans(fs, w, s):
        seen.add(kind)
        tag = "%s kernel, fs=%d w=%d s=%d" % (KIND_NAMES[kind], fs, w, s)
        out = P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl)
        out34 = P.feature_extraction_batch(d, fs, w, s, lengths=lens, plan=pl, deltas=False).cpu().numpy()
        got = out.cpu().numpy()
        for i, name in enumerate(names):
            check_clip(got[i, :, :T[i]], refs[i], K, kind, name, "%s: %s" % (tag, name), True)
            check_clip(out34[i, :, :T[i]], refs[i][:34], K, kind, name, "%s, no deltas: %s" % (tag, name), True)
            assert not got[i, :, T[i]:].any()
            da, la = ragged([clips[i]], np.int16)
            alone = P.feature_extraction_batch(da, fs, w, s, lengths=la, plan=pl)
            if kind == CTA:         # alone, the row stride is the clip's length: another staging variant unless it is a multiple of 8
                check_clip(alone[0].cpu().numpy(), refs[i], K, kind, name, "%s alone: %s" % (tag, name), True)
            else:
                assert torch.equal(alone[0], out[i, :, :T[i]]), "%s: %s alone differs from the batch" % (tag, name)
        oodd = P.feature_extraction_batch(dodd, fs, w, s, lengths=lens, plan=pl)
        if kind == CTA:
            godd = oodd.cpu().numpy()
            for i, name in enumerate(names):
                check_clip(godd[i, :, :T[i]], refs[i], K, kind, name, "%s, odd offset: %s" % (tag, name), True)
        else:
            for i, name in enumerate(names):
                assert torch.equal(oodd[i, :, :T[i]], out[i, :, :T[i]]), "%s: %s, the odd-offset view differs from the aligned batch" % (tag, name)
        gf = P.feature_extraction_batch(df, fs, w, s, lengths=flens, plan=pl).cpu().numpy()
        for i, name in enumerate(fnames):
            check_clip(gf[i, :, :frefs[i].shape[1]], frefs[i], K, kind, name, "%s: %s" % (tag, name), False)
    assert seen == kinds, (seen, kinds)


@pytest.mark.parametrize("fs,w,s", ROW_CONFIGS, ids=["%d-%d-%d" % c for c in ROW_CONFIGS])
def test_rows_every_kernel(P, fs, w, s):
    """spectrogram / chromagram rows through the default, CTA, solo and generic kernels (the row kinds have no lengths
    argument: the bank is cut to its shortest clip)."""
    import torch
    ints = SG.bank(fs, w, s)
    flts = SG.float_bank(fs, w, s)
    for bank, dtype in ((ints, np.int16), (flts, np.float32)):
        n = min(x.size for x in bank.values())
        clips = np.stack([x[:n] for x in bank.values()])
        d = torch.from_numpy(clips).cuda()
        xs = [c.astype(np.float64) if dtype == np.float32 else c for c in clips]
        ch_ref = [O.chromagram(x, fs, w, s)[0] for x in xs]
        for kind, pl in plans(fs, w, s):
            if kind == PAIR:
                continue                      # the pair kernel has no row mode: the CTA kernel serves these rows
            sp = P.spectrogram_batch(d, fs, w, s, plan=pl).cpu().numpy()
            ch = P.chromagram_batch(d, fs, w, s, plan=pl).cpu().numpy()
            for i, name in enumerate(bank):
                what = "%s rows, fs=%d w=%d s=%d: %s" % (KIND_NAMES[kind], fs, w, s, name)
                check_spectrogram_rows(sp[i], clips[i], w, s, "spectrogram " + what)
                check_close(ch[i], ch_ref[i], "chromagram " + what, atol=1e-6)

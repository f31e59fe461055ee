"""Helpers shared by the GPU test modules: the kernel kinds a plan reaches and ragged batches on the device."""
import numpy as np

PAIR, SOLO, CTA, GENERIC = 2, 3, 1, 0
KIND_NAMES = {PAIR: "pair", SOLO: "solo", CTA: "CTA", GENERIC: "generic"}


def plans(fs, w, s):
    """[(kind, Plan)] for every kernel kind a plan for (fs, w, s) reaches, the default choice first."""
    from pyaudioanalysis_b200._lib import Plan
    out = [(Plan(fs, w, s).kernel_kind(), Plan(fs, w, s))]
    for kind in (PAIR, SOLO, CTA):
        pl = Plan(fs, w, s).prefer_kernel(kind)
        if pl.kernel_kind() == kind:
            out.append((kind, pl))
    pg = Plan(fs, w, s)
    pg.force_generic(True)
    assert pg.kernel_kind() == GENERIC
    out.append((GENERIC, pg))
    return out


def ragged(clips, dtype, offset=0, pad=0):
    """[B, Nmax] CUDA batch of the clips and their lengths; samples past a clip's length are ``pad``.  offset 0: a view
    of a buffer with 16-byte aligned rows (a row stride that is a multiple of 8 samples); offset > 0: a view into a wider
    buffer whose rows start ``offset`` samples in and whose row stride is not a multiple of 8 samples.  ``pad`` may be
    an array: it is tiled over each row's padding."""
    import torch
    n = max(x.size for x in clips)
    width = -(-(n + offset) // 8) * 8 + (1 if offset else 0)
    buf = np.empty((len(clips), width), dtype=dtype)
    fill = np.resize(np.asarray(pad, dtype=dtype), width)
    for i, x in enumerate(clips):
        buf[i] = fill
        buf[i, offset:offset + x.size] = x
    d = torch.from_numpy(buf).cuda()[:, offset:offset + n]
    lens = torch.tensor([x.size for x in clips], dtype=torch.int64, device="cuda")
    return d, lens

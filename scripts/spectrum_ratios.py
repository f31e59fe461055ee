"""Worst measured err / bound of the spectrum check per kernel kind and window class (DESIGN section 6), and what the
x - x[frame start] subtraction costs on the frames of edge_impulses_f32 at 800 / 200 (a loud first sample).  Runs the
cases of tests/test_gpu_spectra.py through its helpers; any case outside the bound raises.

    python scripts/spectrum_ratios.py        (on a GPU machine)
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from oracle import st_oracle as O
    from tests import parity as PA
    from tests import signals as SG
    from tests import test_gpu_spectra as TS
    from tests.kernels import CTA, GENERIC_SWEEP, KIND_NAMES, PAIR, SOLO, plans
    from pyaudioanalysis_b200._lib import Plan
    import pyaudioanalysis_b200 as pkg
    worst = {}

    def note(kind, cls, ratios):
        r = worst.get((kind, cls), (0.0, 0.0))
        worst[(kind, cls)] = (max([r[0]] + [q[0] for q in ratios]), max([r[1]] + [q[1] for q in ratios]))

    for fs, w, s in TS.PAIR_CONFIGS:
        note("pair", "hop N/2" if 2 * s == w else "other hops", TS.pair_spectra(pkg, fs, w, s))
    for kind, configs in ((SOLO, TS.SOLO_CONFIGS), (CTA, TS.CTA_CONFIGS)):
        for fs, w, s in configs:
            for cls, ratios in TS.row_spectra(pkg, Plan(fs, w, s).prefer_kernel(kind), fs, w, s, KIND_NAMES[kind],
                                              offset_view=kind == CTA).items():
                note(KIND_NAMES[kind], cls, ratios)
    for fs, w, G, path in GENERIC_SWEEP:
        cls = "%s, %s" % ("even" if w % 2 == 0 else "odd", "global scratch" if G == 0 else "G = %d" % G)
        note("generic", cls, TS.generic_spectra(pkg, fs, w, path))
    for (kind, cls), (r, rd) in sorted(worst.items()):
        print(json.dumps({"kernel": kind, "class": cls, "bins_err_over_bound": round(r, 4), "dc_err_over_bound": round(rd, 4)}))
    # edge_impulses_f32 at 800 / 200: err / bound with |z| (the check) and with |y_frame| in its place (a transform of
    # y itself), and the largest |z| / |y_frame|
    fs, w, s = 16000, 800, 200
    x = SG.float_bank(fs, w, s)["edge_impulses_f32"]
    d = torch.from_numpy(x).cuda()[None]
    starts = np.arange(w, len(x) - w + 1, s)
    ref, bins, _, _ = PA.spectrum_reference(x, starts, w)
    y = O.normalize_clip(x.astype(np.float64))
    fr = np.stack([y[a:a + w] for a in starts])
    grow = np.linalg.norm(fr - fr[:, :1], axis=1) / np.linalg.norm(fr, axis=1)
    for kind, pl in plans(fs, w, s):
        if kind == PAIR:
            continue
        got = pkg.spectrogram_batch(d, fs, w, s, plan=pl)[0].cpu().numpy()[:len(starts)].astype(np.float64)
        e = np.linalg.norm(got[:, 1:] - ref[:, 1:], axis=1)
        old_tol = 1e-4 * (np.abs(ref) + 0.1 * np.abs(ref).max(axis=1, keepdims=True)) + 1e-12
        print(json.dumps({"edge_impulses_f32_800_200": KIND_NAMES[kind], "max_err_over_bound": float((e / bins).max()),
                          "max_err_over_bound_with_y_norm": float((e / (bins / grow)).max()),
                          "max_z_over_y_norm": float(grow.max()),
                          "old_per_bin_check_misses": int((np.abs(got - ref) > old_tol).sum())}))


if __name__ == "__main__":
    main()

"""Diagnostics for the warp-autonomous pair kernel (csrc/pair_kernel.cuh) on a GPU box: per-row error against the
oracle for every window it covers, against the other kernels, and a timing of BASELINE configs[1] per kernel kind.

    python scripts/pair_check.py | tee pair_check.log
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pyaudioanalysis_b200 as pkg                      # noqa: E402
from pyaudioanalysis_b200._lib import Plan             # noqa: E402
from oracle import st_oracle as O                      # noqa: E402  (checker only)
from tests import signals as SG                        # noqa: E402

NAMES = O.feature_names(True)


def report(tag, got, ref, K):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    if got.shape != ref.shape:
        print("%-44s SHAPE %s vs %s" % (tag, got.shape, ref.shape))
        return False
    err = np.abs(got - ref)
    tol = 1e-4 * np.abs(ref) + 1e-5
    ratio = err / tol
    ratio[~np.isfinite(got)] = np.inf
    worst = ratio.max(axis=1)
    bad = [(NAMES[r] if r < len(NAMES) else str(r), float(worst[r]), int((ratio[r] > 1).sum())) for r in np.argsort(-worst)[:6] if worst[r] > 1]
    # rolloff rows may flip by one quantum
    bad = [b for b in bad if not (b[0].endswith("spectral_rolloff") and err[NAMES.index(b[0])].max() <= 2.0 / K + 1e-6)]
    print("%-44s %s  max err/tol %.2f %s" % (tag, "ok " if not bad else "BAD", float(np.nanmax(worst[np.isfinite(worst)])) if np.isfinite(worst).any() else -1, bad))
    return not bad


def main():
    torch.cuda.set_device(0)
    ok = True
    cases = [(16000, 800, 400, 48000), (16000, 800, 400, 32400), (16000, 800, 200, 20000), (16000, 800, 800, 24000), (16000, 800, 333, 20000),
             (16000, 320, 160, 12000), (16000, 480, 240, 14000), (16000, 640, 320, 20000), (16000, 640, 160, 12000),
             (16000, 960, 480, 30000), (48000, 960, 960, 40000), (16000, 1024, 512, 30000), (16000, 512, 256, 20000), (16000, 1024, 256, 20000), (8000, 320, 80, 8000), (16000, 800, 400, 800), (16000, 800, 400, 1200),
             (44100, 882, 441, 50000), (44100, 882, 882, 30000), (44100, 882, 300, 20000), (16000, 400, 160, 20000), (16000, 400, 200, 12000),
             (8000, 600, 300, 12000), (44100, 882, 441, 882), (44100, 882, 441, 1323)]
    for fs, w, s, n in cases:
        x = O.synth_clip(100 + w + s, n, fs)
        ref = O.feature_extraction(x, fs, w, s)[0]
        d = torch.from_numpy(x).cuda()[None]
        for kind in (2, 3, 1, 0):
            pl = Plan(fs, w, s).prefer_kernel(kind)
            if pl.kernel_kind() != kind:
                continue
            got = pkg.feature_extraction_batch(d, fs, w, s, plan=pl)[0].cpu().numpy()
            ok &= report("fs=%d w=%d s=%d n=%d kernel %d(%d)" % (fs, w, s, n, kind, pl.kernel_kind()), got, ref, w // 2)
    # the adversarial signal bank of the test suite (tests/signals.py), int16 and float32
    bank = dict(SG.bank(16000, 800, 400))
    bank.update(SG.float_bank(16000, 800, 400))
    for name, xx in bank.items():
        ref = SG.patch_noise_defined(O.feature_extraction(xx.astype(np.float64) if xx.dtype == np.float32 else xx, 16000, 800, 400)[0],
                                     xx, 800, 400)[0]
        d = torch.from_numpy(xx).cuda()[None]
        for kind in (2, 1):
            got = pkg.feature_extraction_batch(d, 16000, 800, 400, plan=Plan(16000, 800, 400).prefer_kernel(kind))[0].cpu().numpy()
            ok &= report("%s kernel %d" % (name, kind), got, ref, 400)
    # batch / ragged / split independence
    clips = np.stack([O.synth_clip(i, 32000, 16000) for i in range(5)])
    d = torch.from_numpy(clips).cuda()
    p2 = Plan(16000, 800, 400).prefer_kernel(2)
    out = pkg.feature_extraction_batch(d, 16000, 800, 400, plan=p2)
    alone = pkg.feature_extraction_batch(d[2:3], 16000, 800, 400, plan=p2)
    print("split independence (bit-exact):", bool(torch.equal(alone[0], out[2])))
    big = torch.from_numpy(np.stack([O.synth_clip(i % 7, 160000, 16000) for i in range(300)])).cuda()
    ob = pkg.feature_extraction_batch(big, 16000, 800, 400, plan=p2)
    print("long-run vs short-run segmentation (bit-exact):", bool(torch.equal(ob[7], ob[0])), bool(torch.equal(ob[7 + 7 * 20], ob[0])))
    ok &= report("clip 0 of a 300-clip batch", ob[0].cpu().numpy(), O.feature_extraction(O.synth_clip(0, 160000, 16000), 16000, 800, 400)[0], 400)
    lens = torch.tensor([32000, 800, 12345, 31999, 20000], dtype=torch.int64, device="cuda")
    outr = pkg.feature_extraction_batch(d, 16000, 800, 400, lengths=lens, plan=p2)
    for i, L in enumerate(lens.tolist()):
        ref = O.feature_extraction(clips[i][:L], 16000, 800, 400)[0]
        ok &= report("ragged clip %d len %d" % (i, L), outr[i].cpu().numpy()[:, :ref.shape[1]], ref, 400)
    # timing: BASELINE configs[1] per kernel kind
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    c2 = (3000.0 * torch.randn((1000, 160000), generator=g, device="cuda")).round().clamp(-32768, 32767).to(torch.int16)
    out = torch.empty((1000, 68, 399), device="cuda")
    norm = pkg.clip_stats(c2)
    for kind, env in ((1, None), (2, None), (2, "40,8"), (2, "28,12"), (2, "64,8"), (2, "20,5"), (2, "100,10")):
        if env:
            os.environ["B200AA_PAIR_SEG"] = env
        else:
            os.environ.pop("B200AA_PAIR_SEG", None)
        pl = Plan(16000, 800, 400).prefer_kernel(kind)
        for _ in range(3):
            pkg.feature_extraction_batch(c2, 16000, 800, 400, out=out, norm=norm, plan=pl)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            pkg.feature_extraction_batch(c2, 16000, 800, 400, out=out, norm=norm, plan=pl)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        print(json.dumps({"kernel": kind, "seg": env, "ms": ms, "Mframes_per_s": 399000 / ms / 1e3}))
    os.environ.pop("B200AA_PAIR_SEG", None)
    for w, s_ in ((1024, 512), (512, 256), (400, 160), (400, 200)):
        T = (160000 - w) // s_ + 1
        o2 = torch.empty((1000, 68, T), device="cuda")
        for kind in (2, 3, 1):
            pl = Plan(16000, w, s_).prefer_kernel(kind)
            if pl.kernel_kind() != kind:
                continue
            for _ in range(2):
                pkg.feature_extraction_batch(c2, 16000, w, s_, out=o2, norm=norm, plan=pl)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                pkg.feature_extraction_batch(c2, 16000, w, s_, out=o2, norm=norm, plan=pl)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            print(json.dumps({"window": w, "step": s_, "kernel": pl.kernel_kind(), "ms": ms, "Mframes_per_s": 1000 * T / ms / 1e3}))
    # config 3 shape: 16 x 60 s @44.1 kHz, 882 / 441, per kernel kind and mode
    c3 = (3000.0 * torch.randn((16, 2646000), generator=g, device="cuda")).round().clamp(-32768, 32767).to(torch.int16)
    for kind in (3, 1):
        pl = Plan(44100, 882, 441).prefer_kernel(kind)
        row = {"config3_kernel": pl.kernel_kind()}
        for name, fn in (("features", lambda: pkg.feature_extraction_batch(c3, 44100, 882, 441, plan=pl)),
                         ("spectrogram", lambda: pkg.spectrogram_batch(c3, 44100, 882, 441, plan=pl)),
                         ("chromagram", lambda: pkg.chromagram_batch(c3, 44100, 882, 441, plan=pl))):
            fn(); fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 3
            row[name + "_ms"] = ms
            row[name + "_Mrows_per_s"] = 16 * 5999 / ms / 1e3
        print(json.dumps(row))
    print("ALL OK" if ok else "SOME BAD")


if __name__ == "__main__":
    main()

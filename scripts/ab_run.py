"""A/B several builds of libb200aa.so in one process tree: quick parity against the oracle + kernel timing per build.

    python scripts/build_variants.py p2x8 mb4                      # no GPU needed
    python scripts/ab_run.py default p2x8 mb4                      # on the GPU

Every build runs in its own process (the library is chosen at import time through B200AA_LIB).  Prints one JSON line
per build: {"lib", "parity_ok", "worst", "kernel_ms" (median of 20 launches, CUDA events around the fused kernel only),
"frames_per_s", "host_call_ms" / "host_call_frames_per_s" (b200aa_st_features_host on pinned host buffers, 1000 clips),
"host_call_matches_device"}.  This is a development tool: bench.py stays the number of record.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def one():
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import bench
    import pyaudioanalysis_b200 as pkg
    from oracle import st_oracle as O
    from tests.parity import check_features
    res = {"lib": os.environ.get("B200AA_LIB") or "default", "parity_ok": True, "worst": ""}
    # ---- parity: the bench shape and two other register-tiled shapes, ragged tail included
    for fs, w, s, n in ((16000, 800, 400, 48000), (16000, 400, 160, 20000), (16000, 640, 320, 20000), (44100, 882, 441, 30000)):
        clips = np.stack([O.synth_clip(7 * i + w, n, fs) for i in range(5)])
        out = pkg.feature_extraction_batch(torch.from_numpy(clips).cuda(), fs, w, s).cpu().numpy()
        for i in range(5):
            try:
                check_features(out[i], O.feature_extraction(clips[i], fs, w, s)[0], w // 2, "%d/%d clip %d" % (w, s, i))
            except AssertionError as exc:
                res["parity_ok"] = False
                res["worst"] = str(exc)[:300]
    # ---- timing on the bench workload
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    clips = torch.randint(-12000, 12000, (bench.CLIPS_PER_GPU, bench.CLIP_SAMPLES), generator=g, device="cuda", dtype=torch.int16)
    plan = pkg._lib.get_plan(bench.FS, bench.WINDOW, bench.STEP)
    norm = pkg.clip_stats(clips)
    out = None
    for _ in range(3):
        out = pkg.feature_extraction_batch(clips, bench.FS, bench.WINDOW, bench.STEP, norm=norm, out=out, plan=plan)
    times = []
    for _ in range(20):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        pkg.feature_extraction_batch(clips, bench.FS, bench.WINDOW, bench.STEP, norm=norm, out=out, plan=plan)
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    res["kernel_ms"] = times[len(times) // 2]
    res["kernel_ms_min"] = times[0]
    res["frames_per_s"] = bench.CLIPS_PER_GPU * bench.FRAMES_PER_CLIP / (res["kernel_ms"] * 1e-3)
    # ---- other shapes (kernel only): config 3's features (solo kernel) and other pair-kernel windows on the bench batch
    def kernel_ms(c, fs, w, st_, reps=7):
        nrm = pkg.clip_stats(c)
        o = None
        for _ in range(2):
            o = pkg.feature_extraction_batch(c, fs, w, st_, norm=nrm, out=o)
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            pkg.feature_extraction_batch(c, fs, w, st_, norm=nrm, out=o)
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        ts.sort()
        return ts[len(ts) // 2]
    if os.environ.get("B200AA_AB_MORE"):
        res["other_windows_ms"] = {"%d/%d" % (w, st_): kernel_ms(clips, 16000, w, st_) for w, st_ in ((1024, 512), (640, 320), (512, 256), (320, 160), (400, 160))}
        c3 = torch.randint(-12000, 12000, (64, 2646000), generator=g, device="cuda", dtype=torch.int16)
        res["config3_features_ms"] = kernel_ms(c3, 44100, 882, 441, reps=5)
        res["config3_frames_per_s"] = 64 * 5999 / (res["config3_features_ms"] * 1e-3)
        del c3
    # ---- end to end through the C ABI's host entry point (pinned host buffers, copies inside the timed region)
    import ctypes
    import time
    h_in = torch.empty((bench.CLIPS_PER_GPU, bench.CLIP_SAMPLES), dtype=torch.int16).pin_memory()
    h_in.copy_(clips)
    h_out = torch.empty((bench.CLIPS_PER_GPU, 68, bench.FRAMES_PER_CLIP), dtype=torch.float32).pin_memory()
    L = pkg._lib.lib()
    call = lambda: pkg._lib.check(L.b200aa_st_features_host(plan.handle, ctypes.c_void_p(h_in.data_ptr()), 0, bench.CLIPS_PER_GPU,
                                                            bench.CLIP_SAMPLES, 1, ctypes.c_void_p(h_out.data_ptr())))
    call()
    t0 = time.perf_counter()
    for _ in range(5):
        call()
    res["host_call_ms"] = 1e3 * (time.perf_counter() - t0) / 5
    res["host_call_frames_per_s"] = bench.CLIPS_PER_GPU * bench.FRAMES_PER_CLIP / (res["host_call_ms"] * 1e-3)
    res["host_call_matches_device"] = bool(torch.equal(h_out[:8], out[:8].cpu()) and torch.equal(h_out[-8:], out[-8:].cpu()))
    print(json.dumps(res), flush=True)


def main(names):
    for name in names or ["default"]:
        env = dict(os.environ)
        env.pop("B200AA_LIB", None)
        if name != "default":
            path = name if os.path.isabs(name) else os.path.join(ROOT, "pyaudioanalysis_b200", "variants", "libb200aa_%s.so" % name)
            if not os.path.exists(path):
                print(json.dumps({"lib": name, "error": "not built: " + path}), flush=True)
                continue
            env["B200AA_LIB"] = path
        try:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one"], env=env, capture_output=True, text=True, timeout=240)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            print(line[-1] if line else json.dumps({"lib": name, "error": (r.stderr or r.stdout)[-400:]}), flush=True)
        except subprocess.TimeoutExpired:
            print(json.dumps({"lib": name, "error": "timeout (240 s)"}), flush=True)


if __name__ == "__main__":
    if "--one" in sys.argv:
        one()
    else:
        main([a for a in sys.argv[1:] if not a.startswith("-")])

"""GPU: every entry of kernel 12's 68 feature rows under the float64 bound of ``f64_bounds.feature_bounds64``, every frame
included (constant frames and the deltas after them too), and the feature stage restated on the kernel's own spectra.

* Bound: SG.bank (int16), SG.float_bank (float32), the bank as float64 values float32 cannot hold (``kind_clip``'s
  transform), clips whose samples are all equal and ``SG.odd_tail``, each dtype one ragged batch into poisoned output,
  deltas on and off, at every ``kernels.FEATURE_CONFIGS`` entry; ``kind_clip`` at every window of ``f64_bounds.SWEEP``
  whose features the oracle computes (both sides of the shared-memory cap among them), the oracle's refusals elsewhere.
* Stage identity (windows the hop divides): spectrogram row r is feature frame w / s + r; rows 3, 4, 6, 7, 21 .. 33
  equal the stage model of those spectra bit for bit, rows 2, 5, 8 .. 20 within CUDA's log error.
* Deltas: the kernel's own row differences bit for bit, column 0 zero, in every clip of a ragged batch.
* Clips whose samples are all equal normalise to y == 0: every row equals the reference's value exactly, the MFCCs
  within the DCT stage margin.
One JSON line per config: the worst err / bound per row group and the unbounded entries per reason."""
import json

import numpy as np
import pytest
import torch

from oracle import st_oracle as O
from pyaudioanalysis_b200 import batch as BT
from tests import f64_bounds as FB
from tests import host_exe
from tests import signals as SG
from tests.host_exe import bits
from tests.kernels import FEATURE_CONFIGS, ragged

pytestmark = pytest.mark.gpu

F64 = torch.float64
POISON = 0x7ff4dead0000beef
GROUPS = {"time": (0, 1, 2), "spectral": (3, 4, 5, 6, 7), "mfcc": tuple(range(8, 21)), "chroma": tuple(range(21, 34)),
          "deltas": tuple(range(34, 68))}
CONFIGS = [c[:3] for c in FEATURE_CONFIGS]
# unbounded entries (a denominator's interval reaching 0) expected per config: none on these inputs
UNBOUNDED = {c: 0 for c in CONFIGS}


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "f64_host.cu", "-O2")


def dev(x):
    return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def f64_bank(fs, w, s):
    """The int16 bank as float64 values float32 cannot hold: x * 1.000123e-3 + 0.25 + 1e-9 noise."""
    rng = np.random.default_rng(w + 7 * s)
    return {k + "_f64": x * 1.000123e-3 + 0.25 + 1e-9 * rng.normal(size=x.size) for k, x in SG.bank(fs, w, s).items()}


def equal_clips(fs):
    return {"zeros": np.zeros(fs + 3, np.int16), "const_1234": np.full(fs + 29, 1234, np.int16)}


def batch(xs, dtype, fs, w, s, deltas):
    d, L = ragged(xs, dtype)
    B, N = d.shape
    T = O.frame_count(N, w, s)
    out = torch.full((B, 68 if deltas else 34, T), 0, dtype=torch.int64, device="cuda").fill_(POISON).view(F64)
    F = BT.feature_extraction_batch(d, fs, w, s, deltas=deltas, lengths=L, out=out, dtype=F64).cpu().numpy()
    return F, d, L


def note(acc, worst, unb):
    for k, v in worst.items():
        acc["worst"][k] = max(acc["worst"].get(k, 0.0), v)
    for k, v in unb.items():
        acc["unbounded"][k] = acc["unbounded"].get(k, 0) + v


def check_equal_clip(F, x, fs, w, s, what):
    """A clip of equal samples: y == 0, every spectrum exactly 0; each row the reference's exact value, the MFCCs
    D @ log10(eps) within the DCT stage margin."""
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    assert not y.any()
    T = O.frame_count(x.size, w, s)
    ref = O.feature_extraction_loop(x, fs, w, s, tables_per_frame=False)[0]
    mf = list(range(8, 21)) + list(range(42, 55))
    other = [r for r in range(68) if r not in mf]
    assert (F[other, :T] == ref[other]).all(), what
    lm = abs(np.log10(FB.EPS))
    margin = 2 * float(FB.gamma64(41)) * lm * np.abs(O.dct_matrix()).sum(axis=1)
    assert (np.abs(F[8:21, :T] - ref[8:21]) <= margin[:, None]).all(), what
    assert not F[42:55, :T].any() and not F[[3, 4, 5, 6, 7, 21], :T].any(), what


def check_clip(F, Fnd, x, fs, w, s, what, acc, sp=None, tables=None):
    """Clip x's block F [68, >= T] (deltas) and Fnd [34, >= T] (no deltas) of a ragged batch: the bound, the deltas, the
    rows without deltas equal, padding poisoned; with sp (the clip's spectrogram rows) the stage identity."""
    T = O.frame_count(x.size, w, s)
    assert (F[:, T:].view(np.int64) == POISON).all() and (Fnd[:, T:].view(np.int64) == POISON).all(), what + ": padding"
    assert (bits(Fnd[:, :T]) == bits(F[:34, :T])).all(), what + ": rows without deltas differ"
    FB.check_deltas(F, T, what)
    fb = FB.feature_bounds64(x, fs, w, s, deltas=True)
    worst, unb = FB.check_feature_bounds64(F[:, :T], fb, what)
    note(acc, worst, unb)
    sel = np.abs(fb.ref) > 0
    for g, rows in GROUPS.items():
        rr = [r for r in rows if r != 7 and r != 41]
        m = sel[rr] & np.isfinite(fb.bound[rr])
        if m.any():
            acc["median_rel"].setdefault(g, []).append(float(np.median((fb.bound[rr] / np.where(sel[rr], np.abs(fb.ref[rr]), 1))[m])))
    if sp is not None and w % s == 0:
        r0 = w // s
        R = min(sp.shape[0], T - r0)
        if R > 0:
            y = O.normalize_clip(np.asarray(x, dtype=np.float64))
            fr = np.stack([y[s * t:s * t + w] for t in range(r0, r0 + R)])
            X = sp[:R]
            Xp = np.concatenate([X[:1], X[:-1]])
            st = FB.stage_model(X, Xp, fs, *tables, frames=fr)
            got = F[:34, r0:r0 + R]
            acc["log margin"] = max(acc.get("log margin", 0.0), FB.check_stage(got, st, what + " stage",
                                                                               [r for r in range(34) if r != 6]))
            if R > 1:
                FB.check_stage(got[:, 1:], FB.Stage(st.rows[:, 1:], st.margin[:, 1:], st.have), what + " stage flux", [6])
            acc["stage frames"] = acc.get("stage frames", 0) + R
    return fb


@pytest.mark.parametrize("fs,w,s", CONFIGS, ids=["%d-%d-%d" % c for c in CONFIGS])
def test_feature_configs(harness, fs, w, s):
    acc = {"worst": {}, "unbounded": {}, "median_rel": {}}
    tables = FB.stage_tables(harness, fs, w // 2)
    groups = {np.int16: {**SG.bank(fs, w, s), **equal_clips(fs), "odd_tail": SG.odd_tail(fs, w, s)},
              np.float32: SG.float_bank(fs, w, s), np.float64: f64_bank(fs, w, s)}
    for dtype, clips in groups.items():
        names, xs = list(clips), list(clips.values())
        F, d, L = batch(xs, dtype, fs, w, s, True)
        Fnd, _, _ = batch(xs, dtype, fs, w, s, False)
        sp = BT.spectrogram_batch(d, fs, w, s, lengths=L, dtype=F64).cpu().numpy() if w % s == 0 else None
        counts = BT.row_counts(L, w, s, 0).cpu().tolist()
        for i, (name, x) in enumerate(zip(names, xs)):
            what = "%d/%d/%d %s" % (fs, w, s, name)
            check_clip(F[i], Fnd[i], x, fs, w, s, what, acc, None if sp is None else sp[i, :counts[i]], tables)
            if name in ("zeros", "const_1234"):
                check_equal_clip(F[i], x, fs, w, s, what)
    assert sum(acc["unbounded"].values()) == UNBOUNDED[(fs, w, s)], acc["unbounded"]
    acc["median_rel"] = {k: float(np.median(v)) for k, v in acc["median_rel"].items()}
    print(json.dumps({"config": [fs, w, s], **acc}))


def sweep_fs(w):
    return 44100 if w in (882, 2205, 44100, FB.SMEM_LAST, FB.BIG_FIRST) else 16000


def oracle_refusal(x, fs, w):
    """The exception type with which the oracle refuses the window, or None."""
    try:
        O.feature_extraction(x, fs, w, w)
        return None
    except (ValueError, IndexError) as exc:
        return type(exc)


@pytest.mark.parametrize("w", FB.SWEEP)
def test_window_sweep(harness, w):
    fs = sweep_fs(w)
    acc = {"worst": {}, "unbounded": {}, "median_rel": {}}
    for dtype in (np.int16, np.float32, np.float64):
        x = FB.kind_clip(w, dtype)
        refusal = oracle_refusal(x, fs, w)
        if refusal is not None:
            with pytest.raises(refusal):
                BT.feature_extraction_batch(dev(x), fs, w, w, dtype=F64)
            acc["refused"] = True
            continue
        tables = FB.stage_tables(harness, fs, w // 2)
        F, d, L = batch([x], dtype, fs, w, w, True)
        Fnd, _, _ = batch([x], dtype, fs, w, w, False)
        sp = BT.spectrogram_batch(d, fs, w, w, lengths=L, dtype=F64).cpu().numpy()[0]
        n_sp = BT.row_counts(L, w, w, 0).cpu().tolist()[0]
        check_clip(F[0], Fnd[0], x, fs, w, w, "sweep w=%d %s" % (w, np.dtype(dtype).name), acc, sp[:n_sp], tables)
    assert not acc["unbounded"], acc["unbounded"]
    acc["median_rel"] = {k: float(np.median(v)) for k, v in acc["median_rel"].items()}
    print(json.dumps({"w": w, "fs": fs, **acc}))

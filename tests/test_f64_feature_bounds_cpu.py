"""CPU: the float64 feature bound (``f64_bounds.feature_bounds64``) and the stage model (``f64_bounds.stage_model``) of
kernel 12's 68 feature rows.

* The bound holds the oracle's own features computed from spectra perturbed inside the spectrum ball, toward the worst
  direction of each row, on the signal bank, the frame kinds and a clip whose samples are all equal.
* The host build of kernel 12's transform (tests/f64_host.cu) through the stage model lands inside the bound at every
  window of ``f64_bounds.SWEEP`` whose features the oracle computes.
* Planted defects pass ``assert_allclose(rtol=1e-9, atol=1e-11)`` on the frames the float64 path's oracle tests look at
  (they skip constant frames and the deltas after them), and the bound or the stage identity rejects them."""
import numpy as np
import pytest

from oracle import st_oracle as O
from tests import f64_bounds as FB
from tests import host_exe
from tests import signals as SG
from tests.host_exe import floats, hexes, run

RT, AT = 1e-9, 1e-11


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "f64_host.cu", "-O2")


def host_spec(exe, frames):
    frames = np.asarray(frames, dtype=np.float64)
    out = run(exe, "".join("spec %d %s\n" % (frames.shape[1], hexes(f)) for f in frames))
    return np.stack([floats(line[1:]) for line in out])


def frames_of(x, w, s):
    y = O.normalize_clip(np.asarray(x, dtype=np.float64))
    return np.stack([y[s * t:s * t + w] for t in range(O.frame_count(y.size, w, s))])


def features(X, fr, fs, tables, prev=None):
    """Rows 0 .. 33 from spectra X through the stage model (rows 0 .. 1 from the samples, as the oracle computes them)."""
    Xp = np.concatenate([X[:1], X[:-1]]) if prev is None else prev
    st = FB.stage_model(X, Xp, fs, *tables, frames=fr)
    rows = st.rows.copy()
    rows[0] = [O._zcr(f) for f in fr]
    rows[1] = [O._energy(f) for f in fr]
    return rows


def with_deltas(rows):
    d = np.zeros_like(rows)
    d[:, 1:] = rows[:, 1:] - rows[:, :-1]
    return np.concatenate([rows, d])


def test_host_tables_are_the_oracles(exe):
    """The mel bank and DCT the plan builds are the oracle's bit for bit, so the stage model may use either."""
    for fs, K in ((16000, 400), (44100, 441), (8000, 300), (22050, 275)):
        mel, dct = FB.stage_tables(exe, fs, K)
        M, D, _ = FB._tables(fs, K)
        assert (mel == M).all() and (dct == D).all(), (fs, K)


def directions(X, e, fs, row_ref, M):
    """Unit directions [T, K] toward each row's worst change: the centroid's and the spread's gradients, the first
    entropy block, the whole spectrum up and down, and the smallest non-empty mel band down."""
    T, K = X.shape
    ind = np.arange(1, K + 1) * (fs / (2.0 * K))
    c = row_ref[3] * fs / 2.0
    V = (row_ref[4] * fs / 2.0) ** 2
    blk = max(K // 10, 1)
    B = np.zeros(K)
    B[:blk] = 1.0
    m = X @ M.T
    band = np.argmin(np.where(M.any(axis=1)[None, :], m, np.inf), axis=1)
    out = [ind[None, :] - c[:, None], (ind[None, :] - c[:, None]) ** 2 - V[:, None], (B[None, :] - 0.1) * (X + 1e-300),
           X + 1e-300, -(X + 1e-300), -M[band]]
    res = []
    for d in out:
        d = d + np.where(np.abs(d).sum(axis=1, keepdims=True) == 0, 1.0, 0.0)
        d = d / np.abs(d).max(axis=1, keepdims=True)
        res.append(d / np.linalg.norm(d, axis=1, keepdims=True))
    return res


def clips_for(fs, w, s):
    out = dict(SG.bank(fs, w, s))
    kinds = FB.frame_kinds(w)
    out["kinds"] = np.clip(np.round(np.concatenate([kinds[k] for k in FB.KINDS]) * 30000.0), -32768, 32767).astype(np.int16)
    out["equal"] = np.full(fs // 2 + 7, 1234, np.int16)
    return out


@pytest.mark.parametrize("fs,w,s", [(16000, 800, 400), (44100, 882, 441), (16000, 400, 160)])
def test_bound_holds_the_oracle_inside_the_ball(fs, w, s):
    M, D, _ = FB._tables(fs, w // 2)
    tables = (M, D)
    for name, x in clips_for(fs, w, s).items():
        fb = FB.feature_bounds64(x, fs, w, s, deltas=True)
        fr = frames_of(x, w, s)
        X, e = FB.spectrum_reference(fr)
        assert not fb.unbounded, (name, fb.unbounded)
        for j, d in enumerate(directions(X, e, fs, fb.ref, M)):
            for sign in (1.0, -1.0):
                Xq = np.maximum(X + sign * e[:, None] * d, 0.0)          # the projection stays inside the ball
                got = with_deltas(features(Xq, fr, fs, tables))
                FB.check_feature_bounds64(got, fb, "%s %d/%d/%d, direction %d%+d" % (name, fs, w, s, j, sign))


@pytest.mark.parametrize("w", FB.SWEEP)
def test_host_transform_through_the_stage_within_bound(exe, w):
    fs = 44100 if w in (882, 2205, 44100, FB.SMEM_LAST, FB.BIG_FIRST) else 16000
    x = FB.kind_clip(w, np.int16)
    try:
        O.feature_extraction(x, fs, w, w)
    except (ValueError, IndexError):
        pytest.skip("the oracle refuses w=%d at %d Hz" % (w, fs))
    fr = frames_of(x, w, w)
    got = with_deltas(features(host_spec(exe, fr), fr, fs, FB.stage_tables(exe, fs, w // 2)))
    worst, unb = FB.check_feature_bounds64(got, FB.feature_bounds64(x, fs, w, w, deltas=True), "host w=%d" % w)
    assert not unb
    print("w=%d" % w, {k: "%.3g" % v for k, v in worst.items()})


def test_equal_clip_bound_is_exact():
    """All spectra 0: every bound entry but the MFCCs' is 0, the MFCCs' the DCT stage alone."""
    fs, w, s = 16000, 800, 400
    fb = FB.feature_bounds64(np.full(9000, -77, np.int16), fs, w, s, deltas=True)
    mf = list(range(8, 21)) + list(range(42, 55))
    assert not np.delete(fb.bound, mf, axis=0).any()
    assert (fb.bound[8:21] < 1e-11).all() and (fb.roll == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# planted defects
def old_check_accepts(got, x, fs, w, s):
    """The float64 path's oracle test: rtol 1e-9 / atol 1e-11 against the oracle, constant frames and the deltas of
    the frame after one skipped."""
    ref, _ = O.feature_extraction(x, fs, w, s)
    bad = SG.noise_defined_frames(x, w, s)
    ok = ~bad & ~np.concatenate([[False], bad[:-1]])
    np.testing.assert_allclose(got[:, ok], ref[:, ok], rtol=RT, atol=AT)
    return int(bad.sum())


def tone_clip(fs, w, s):
    """A tone between bins (1000.37 Hz): its spread is small beside its centroid."""
    return np.round(20000.0 * np.sin(2 * np.pi * 1000.37 * np.arange(fs) / fs + 0.3)).astype(np.int16)


def steady_clip(fs, w, s):
    """Noise repeated with period s, 1 LSB added to one sample in a hundred: nearly identical frames, a small flux."""
    rng = np.random.default_rng(11)
    x = np.tile(np.round(rng.normal(0, 3000.0, s)), fs // s)
    return (x + (rng.random(x.size) < 0.01)).astype(np.int16)


def onset_clip(fs, w, s, t0=16):
    """Noise, then the constant 1000 from frame t0 on (frame t0 = 16: the first frame of a work item)."""
    rng = np.random.default_rng(5)
    x = rng.normal(0, 3000.0, fs)
    x[t0 * s:] = 1000.0
    return np.round(x).astype(np.int16)


def spread_one_pass(X, Xp, fr, fs, tables):
    rows = features(X, fr, fs, tables)
    K = X.shape[1]
    ind = np.arange(1, K + 1) * (fs / (2.0 * K))
    top = X.max(axis=1)
    Xt = X / np.where(top == 0, FB.EPS, top)[:, None]
    den = FB.rowsum(Xt) + FB.EPS
    c = FB.rowsum(ind * Xt) / den
    rows[4] = np.sqrt(np.maximum(FB.rowsum(ind ** 2 * Xt) / den - c * c, 0.0)) / (fs / 2.0)
    return rows


def flux_expanded(X, Xp, fr, fs, tables):
    rows = features(X, fr, fs, tables)
    a = X / FB.rowsum(X + FB.EPS)[:, None]
    b = Xp / FB.rowsum(Xp + FB.EPS)[:, None]
    rows[6] = FB.rowsum(a * a) - 2 * FB.rowsum(a * b) + FB.rowsum(b * b)
    return rows


def flux_wrong_previous(X, Xp, fr, fs, tables):
    """At the first frame of every 16-frame work item the frame is taken as its own previous frame."""
    P = Xp.copy()
    P[16::16] = X[16::16]
    return features(X, fr, fs, tables, prev=P)


def entropy_no_eps_total(X, Xp, fr, fs, tables):
    """The spectral entropy's s_j = B_j / total, EPS dropped."""
    rows = features(X, fr, fs, tables)
    Bs, _ = FB._blocks(X)
    with np.errstate(invalid="ignore", divide="ignore"):
        sj = Bs / FB.rowsum(X * X)[:, None]
        rows[5] = -FB.rowsum(sj * FB.cr_log2(sj + FB.EPS))
    return rows


def entropy_eps_1e16(X, Xp, fr, fs, tables):
    """The spectral entropy with 1e-16 in place of EPS in both places."""
    rows = features(X, fr, fs, tables)
    Bs, _ = FB._blocks(X)
    sj = Bs / (FB.rowsum(X * X) + 1e-16)[:, None]
    rows[5] = -FB.rowsum(sj * FB.cr_log2(sj + 1e-16))
    return rows


def nan_in_constant_frames(X, Xp, fr, fs, tables):
    rows = features(X, fr, fs, tables)
    const = (fr == fr[:, :1]).all(axis=1)
    rows[3:34, const] = np.nan
    return rows


# name -> (defect, clip maker (fs, w, s) -> x, the checks that reject it)
BOTH = ["bound", "stage"]
DEFECTS = {
    "one-pass spread, tone": (spread_one_pass, tone_clip, ["stage"]),
    "expanded-square flux, steady frames": (flux_expanded, steady_clip, BOTH),
    "flux previous frame at a work-item start, constant onset": (flux_wrong_previous, onset_clip, BOTH),
    "spectral entropy without EPS in its total, constant onset": (entropy_no_eps_total, onset_clip, BOTH),
    "spectral entropy with 1e-16 for EPS, constant onset": (entropy_eps_1e16, onset_clip, BOTH),
    "NaN in the rows of constant frames": (nan_in_constant_frames, onset_clip, BOTH),
}


@pytest.mark.parametrize("name", list(DEFECTS))
def test_planted_defect_passes_rtol_and_is_rejected(exe, name):
    fs, w, s = 16000, 800, 400
    defect, make, _ = DEFECTS[name]
    x = make(fs, w, s)
    fr = frames_of(x, w, s)
    tables = FB.stage_tables(exe, fs, w // 2)
    X = host_spec(exe, fr)
    Xp = np.concatenate([X[:1], X[:-1]])
    got = with_deltas(defect(X, Xp, fr, fs, tables))
    old_check_accepts(got, x, fs, w, s)
    fb = FB.feature_bounds64(x, fs, w, s, deltas=True)
    FB.check_feature_bounds64(with_deltas(features(X, fr, fs, tables)), fb, name + ", without the defect")
    rejected = []
    for check, call in (("bound", lambda: FB.check_feature_bounds64(got, fb, name)),
                        ("stage", lambda: FB.check_stage(got[:34], FB.stage_model(X, Xp, fs, *tables, frames=fr), name))):
        try:
            call()
        except AssertionError as exc:
            rejected.append(check)
            print(name, "rejected by the", check, "check:", str(exc)[:200])
    assert rejected == DEFECTS[name][2], rejected


def test_rolloff_without_eps_does_not_separate(exe):
    """EPS dropped from the rolloff's comparison changes nothing on the constant onset: its first quantum is the same
    on a zero and on a DC-only spectrum, and a frame with energy has a cumsum far above EPS.  Pinned here so that a
    change of that fact is noticed."""
    fs, w, s = 16000, 800, 400
    x = onset_clip(fs, w, s)
    fr = frames_of(x, w, s)
    tables = FB.stage_tables(exe, fs, w // 2)
    X = host_spec(exe, fr)
    P = np.cumsum(X * X, axis=1)
    tot = FB.rowsum(X * X)
    over = P > (0.90 * tot)[:, None]
    roll = np.where(over.any(axis=1), np.argmax(over, axis=1) / float(w // 2), 0.0)
    assert (roll == features(X, fr, fs, tables)[7]).all()

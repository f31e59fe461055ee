"""CPU: the float64 spectrum and chroma bounds of tests/f64_bounds.py (derivation in its docstring), checked on the host
build of kernel 12's transform (tests/f64_host.cu: ``f64::stockham_output``, its fma calls, the table formula and
``f64::magnitude``, the code the device runs), and shown to reject planted defects that ``assert_allclose(rtol=1e-9,
atol=1e-11)`` -- the float64 path's published contract -- accepts."""
import math

import numpy as np
import pytest

from tests import f64_bounds as FB
from tests import host_exe
from tests.host_exe import floats, hexes, run

RT, AT = 1e-9, 1e-11
COMPOSITE = (800, 882, 2205, 44100)


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "f64_host.cu", "-O2")


def host_spec(exe, frames, cmd="spec"):
    """|X|[0:K] / K of every frame by the host build of kernel 12's transform."""
    frames = np.asarray(frames, dtype=np.float64)
    N = frames.shape[1]
    out = run(exe, "".join("%s %d %s\n" % (cmd, N, hexes(f)) for f in frames))
    return np.stack([floats(line[1:]) for line in out]) if N > 1 else np.zeros((len(frames), 0))


def kinds(N):
    k = FB.frame_kinds(N)
    return [k[n] for n in FB.KINDS]


def test_radices_and_pass_costs():
    assert FB.radices(1) == [] and FB.radices(2) == [2] and FB.radices(8) == [4, 2]
    assert FB.radices(44100) == [4, 3, 3, 5, 5, 7, 7] and FB.radices(20011) == [20011] and FB.radices(1688) == [4, 2, 211]
    # the per-pass costs quoted in the derivation
    for R, c in ((4, 66), (3, 52), (5, 80), (7, 110)):
        assert abs(FB.pass_cost(R) / FB.U64 - c) < 1.5, (R, FB.pass_cost(R) / FB.U64)
    assert 300 < FB.transform_delta(800) / FB.U64 < 360 and 500 < FB.transform_delta(44100) / FB.U64 < 600
    # the shared-memory cap of the frame kernel: f64_warp_bytes (two complex buffers, two |X| rows) against 226 KiB
    warp_bytes = lambda w: (max(w, 20) * 2 * 16 + (w // 2) * 2 * 8 + 15) & ~15
    assert warp_bytes(FB.SMEM_LAST) <= 226 * 1024 < warp_bytes(FB.BIG_FIRST)


@pytest.mark.parametrize("N", FB.SWEEP)
def test_host_transform_within_bound(exe, N):
    """Every frame kind at every window of the sweep: the host build of the transform under the bound."""
    frames = np.stack(kinds(N))
    got = host_spec(exe, frames)
    r = FB.check_spectrum(got, frames, "host transform, N=%d" % N)
    print("N=%d worst err / bound %.4f" % (N, r))


def test_zero_frame_is_exact(exe):
    for N in (2, 9, 882, 997):
        assert not host_spec(exe, np.zeros((1, N))).any()
        FB.check_spectrum(np.zeros((1, N // 2)), np.zeros((1, N)), "zero frame")
        with pytest.raises(AssertionError, match="outside the float64 spectrum bound"):
            FB.check_spectrum(np.full((1, N // 2), 1e-100), np.zeros((1, N)), "zero frame, bins of 1e-100")


@pytest.mark.parametrize("N", COMPOSITE)
def test_one_bin_off_by_1e12_rejected(exe, N):
    frames = np.stack(kinds(N))
    got = host_spec(exe, frames)
    ref, _ = FB.spectrum_reference(frames)
    for kind in ("tone_on_bin", "tone_between_bins"):
        j = FB.KINDS.index(kind)
        k = int(np.argmax(ref[j]))
        bad = got.copy()
        bad[j, k] *= 1 + 1e-12
        np.testing.assert_allclose(bad, ref, rtol=RT, atol=AT)
        with pytest.raises(AssertionError, match="outside the float64 spectrum bound"):
            FB.check_spectrum(bad, frames, "%s, N=%d, bin %d off by 1e-12" % (kind, N, k))


@pytest.mark.parametrize("N", (2205, 20000, 44100))
def test_recurrence_twiddles_rejected(exe, N):
    """Twiddles w^j = w^(j-1) w drift by about j u: inside rtol 1e-9, far outside the bound."""
    frames = np.stack(kinds(N))
    ref, _ = FB.spectrum_reference(frames)
    rec = host_spec(exe, frames, "specrec")
    np.testing.assert_allclose(rec, ref, rtol=RT, atol=AT)
    with pytest.raises(AssertionError, match="outside the float64 spectrum bound"):
        FB.check_spectrum(rec, frames, "recurrence twiddles, N=%d" % N)


def direct_dft(fr, K, f32_twiddles=False):
    """|X|[0:K] / K by a direct DFT over the twiddles sin / cos(pi 2 (j k mod n) / n), kernel 12's clipped-frame form."""
    n = fr.size
    ph = np.outer(np.arange(K), np.arange(n)) % n
    a = np.pi * (2.0 * ph / n)
    c, s = np.cos(a), np.sin(a)
    if f32_twiddles:
        c, s = c.astype(np.float32).astype(np.float64), s.astype(np.float32).astype(np.float64)
    return np.hypot(c @ fr, s @ fr) / K


@pytest.mark.parametrize("w,n", [(800, 400), (800, 401), (800, 797), (882, 661), (5786, 4999)])
def test_clipped_bound(w, n):
    """A direct DFT with fp64 twiddles is inside the per-bin clipped bound; one with float32 twiddles (inside rtol 1e-9
    on the tone's big bins) is not."""
    K = w // 2
    for kind, fr in FB.frame_kinds(n).items():
        X, eps = FB.clipped_reference(fr, K)
        got = direct_dft(fr, K)
        assert (np.abs(got - X) <= eps).all(), (kind, float((np.abs(got - X) / eps).max()))
    fr = FB.frame_kinds(n)["tone_between_bins"]
    X, eps = FB.clipped_reference(fr, K)
    assert (np.abs(direct_dft(fr, K, f32_twiddles=True) - X) > eps).any()


def kernel_chroma(X, fs, K):
    """f64_chroma's order: each class adds X[bin]^2 / share of its taps in ascending slot order, then / sum(X^2)."""
    from oracle import st_oracle as O
    semis, share = O.chroma_tables(fs, K)
    wrap = lambda j: j + K if j < 0 else j
    winner = {}
    for k in range(K):
        winner[wrap(int(semis[k]))] = k
    out = np.zeros((X.shape[0], 12))
    for t, row in enumerate(X):
        tot = float(np.sum(row * row))
        for c in range(12):
            acc = 0.0
            for j in range(c, K, 12):
                if j in winner:
                    acc += row[winner[j]] * row[winner[j]] / share[wrap(int(semis[j]))]
            out[t, c] = acc / (tot if tot != 0 else FB.O_EPS)
    return out


@pytest.mark.parametrize("fs,N", [(16000, 800), (44100, 882), (44100, 2205)])
def test_chroma_of_host_spectra_within_bound(exe, fs, N):
    """The host transform's spectra through the kernel's chroma fold, under chroma_bound64.  A tone on a chroma tap puts
    its class near 1 (the kinds' tones fall on bins whose slot another bin wins: their classes are leakage); that class
    off by 1e-12 relative is rejected."""
    from tests.parity import ROW_FULL, _tables, check_chromagram_bounds
    C = _tables(fs, N // 2)[2]
    tap = int(np.argmax(C.max(axis=0)))
    frames = np.stack(kinds(N) + [np.sin(2 * np.pi * tap * np.arange(N) / N + 0.1)])
    got = kernel_chroma(host_spec(exe, frames), fs, N // 2)
    X, e = FB.spectrum_reference(frames)
    cj = FB._classes(X, C)
    cb = FB.Bounds(cj, FB.chroma_bound64(X, C, cj, e=e), np.full(len(frames), ROW_FULL), False, {})
    worst, unb = check_chromagram_bounds(got, cb, "host chroma, N=%d" % N)
    assert not unb and worst["full"] < 1.0
    c = int(np.argmax(cj[-1]))
    assert cj[-1, c] > 0.3
    bad = got.copy()
    bad[-1, c] *= 1 + 1e-12
    np.testing.assert_allclose(bad[-1], cj[-1], rtol=RT, atol=AT)
    with pytest.raises(AssertionError, match="outside the chromagram bound"):
        check_chromagram_bounds(bad, cb, "planted class")


def test_pairwise_depth():
    assert FB.pairwise_depth(1) == 3 and FB.pairwise_depth(7) == 9
    assert FB.pairwise_depth(128) == 28 and FB.pairwise_depth(129) == 29 and FB.pairwise_depth(22050) == 36
    assert math.isclose(float(FB.gamma64(36)), 36 * FB.U64, rel_tol=1e-12)

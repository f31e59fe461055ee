"""GPU: the last-bit banks of tests/last_bit_cases.py through kernels 5, 6 and 7 -- permuted kNN pairs, cyclic
cross-validation problems, permuted-mean and duplicated-state HMMs, on which one ulp of a distance, a scaler sum or a log
density changes a neighbour, a prediction or a state -- bit for bit against the oracles; and kernel 3
(b200aa_normalize_windows) bit for bit against NumPy's float32 (mid - mean) / std, non-finite values and subnormals
included."""
import types

import numpy as np
import pytest

from tests import knn_cv_oracle
from tests import last_bit_cases as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def C():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from pyaudioanalysis_b200 import consumers
    return consumers


@pytest.fixture(scope="module")
def knn_banks():
    return [(b, L.knn_expected(b)) for b in L.knn_banks()]


def _knn_model(C, bank):
    return C.KnnModel(types.SimpleNamespace(features=bank.feats, labels=bank.labels, neighbors=bank.k))


def _knn_same(C, model, t, ref, what):
    import torch
    ids, P = C.knn_classify_batch(model, t)
    torch.cuda.synchronize()
    assert np.array_equal(ids.cpu().numpy(), ref[0]), what
    assert np.array_equal(P.cpu().numpy(), ref[1]), what


# ------------------------------------------------------------------ kernel 5
def test_knn_permuted_pairs_float64_and_float32(C, knn_banks):
    """k = 1, 2, 7 at F = 1 .. 138: the queries' values are exact in float32, so both widths must give the oracle's."""
    import torch
    for bank, ref in knn_banks:
        model = _knn_model(C, bank)
        q = torch.from_numpy(bank.queries).cuda()
        _knn_same(C, model, q, ref, (bank.F, bank.k, "float64"))
        _knn_same(C, model, q.float(), ref, (bank.F, bank.k, "float32"))


def test_knn_permuted_pairs_strided(C, knn_banks):
    """Query rows read through a row stride wider than F (float64 and float32), and every other row of a buffer."""
    import torch
    for bank, ref in knn_banks:
        model = _knn_model(C, bank)
        n, F = bank.queries.shape
        wide = torch.full((n, F + 7), float("nan"), dtype=torch.float64, device="cuda")
        wide[:, 3:3 + F] = torch.from_numpy(bank.queries).cuda()
        tall = torch.full((2 * n, F), float("nan"), dtype=torch.float64, device="cuda")
        tall[::2] = torch.from_numpy(bank.queries).cuda()
        for t in (wide[:, 3:3 + F], wide.float()[:, 3:3 + F], tall[::2], tall.float()[::2]):
            _knn_same(C, model, t, ref, (bank.F, bank.k, t.dtype, tuple(t.stride())))


def test_knn_permuted_pairs_across_key_slices(C):
    """6 000 queries of 12 000 training rows: 576 MB of keys, three slices of at most 2 796 queries."""
    import torch
    bank = L.knn_bank(77, 16, 1, n_q=6000)
    ref = L.knn_expected(bank)
    _knn_same(C, _knn_model(C, bank), torch.from_numpy(bank.queries).cuda(), ref, "slices")


# ------------------------------------------------------------------ kernel 6
def test_knn_cross_validate_cyclic_problems(C):
    """Eight problems per batch on cyclic training matrices in shuffled split order: predictions and counts."""
    import torch
    for X, y, splits, ks in L.cv_banks():
        pred, counts = C.knn_cross_validate(X, y, splits, ks, 3)
        torch.cuda.synchronize()
        ref = knn_cv_oracle.predict(X, y, splits, ks)
        got = np.split(pred.cpu().numpy(), np.cumsum([len(te) for _, te in splits])[:-1])
        for p, (a, b) in enumerate(zip(got, ref)):
            assert np.array_equal(a, b), p
        assert np.array_equal(counts.cpu().numpy(), knn_cv_oracle.counts(y, splits, ref, 3))


# ------------------------------------------------------------------ kernel 7
COUNTS = [64] * 12 + [1] * 40 + [2, 3, 37, 130]


def _decode(C, t, case):
    import torch
    ids, bad = C.hmm_decode_batch(t, C.HmmModel(case.model), case.counts)
    torch.cuda.synchronize()
    return ids.cpu().numpy(), bad.cpu().numpy()


def _check_paths(case, ids, bad, window_major, what):
    assert not bad.any(), what
    for b, n in enumerate(case.counts):
        assert np.array_equal(ids[b, :n], L.hmm_expected(case, b, window_major)), (what, b, n)
        assert not ids[b, n:].any(), (what, b)


@pytest.mark.parametrize("tie", [False, True])
@pytest.mark.parametrize("n_states", L.HMM_STATES)
def test_hmm_decode_float32_feature_major(C, n_states, tie):
    """A ragged batch (64-window, one-window and other clips, NaN past each count); tie: duplicated states, where the
    tie rule of csrc/hmm.cuh decides every window of a pair."""
    import torch
    case = L.hmm_case(300 + n_states + 1000 * tie, n_states, COUNTS, tie=tie, dtype=np.float32)
    ids, bad = _decode(C, torch.from_numpy(case.x).cuda(), case)
    _check_paths(case, ids, bad, False, (n_states, tie))


@pytest.mark.parametrize("tie", [False, True])
@pytest.mark.parametrize("n_states", L.HMM_STATES)
def test_hmm_decode_float64_both_layouts(C, n_states, tie):
    """Feature-major [B, F, M] (densities in sequence, pairwise for a one-window clip) and the transpose of a
    window-major [B, M, F] batch (pairwise throughout)."""
    import torch
    case = L.hmm_case(400 + n_states + 1000 * tie, n_states, COUNTS, tie=tie)
    ids, bad = _decode(C, torch.from_numpy(case.x).cuda(), case)
    _check_paths(case, ids, bad, False, (n_states, tie, "feature-major"))
    wm = torch.from_numpy(np.ascontiguousarray(case.x.transpose(0, 2, 1))).cuda().transpose(1, 2)
    ids, bad = _decode(C, wm, case)
    _check_paths(case, ids, bad, True, (n_states, tie, "window-major"))


def test_hmm_decode_across_scratch_slices(C):
    """64 states x 12 B per (window, state): 350 004 windows need 269 MB of scratch, so the last clip decodes in a
    second slice."""
    import torch
    case = L.hmm_case(500, 64, [175000, 1, 3, 175000], F=16, dtype=np.float32)
    ids, bad = _decode(C, torch.from_numpy(case.x).cuda(), case)
    _check_paths(case, ids, bad, False, "slices")


# ------------------------------------------------------------------ kernel 3
def _f32_bits(a):
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).copy()
    b[np.isnan(a)] = 0x7fc00000
    return b


def _normalize(C, mid, mean, std):
    import torch
    out = C.normalize_windows_batch(torch.from_numpy(mid).cuda(), mean, std)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _normalize_ref(mid, mean, std):
    return ((mid - mean[None, :, None]) / std[None, :, None]).transpose(0, 2, 1)


@pytest.mark.parametrize("F", [1, 31, 32, 33, 136])
def test_normalize_windows_bit_exact(C, F):
    """Two float32 IEEE operations per value, as NumPy does them: a reciprocal multiply or an FMA would differ."""
    rng = np.random.default_rng(F)
    for M in (1, 31, 32, 33, 4097):
        for B in (1, 3):
            scale = np.float32(10.0) ** rng.uniform(-3, 3, size=(1, F, 1)).astype(np.float32)
            mid = (rng.standard_normal((B, F, M)).astype(np.float32) * scale).astype(np.float32)
            mean = (rng.standard_normal(F) * scale[0, :, 0]).astype(np.float32)
            std = (rng.uniform(0.1, 10.0, size=F) * scale[0, :, 0]).astype(np.float32)
            got = _normalize(C, mid, mean, std)
            assert got.shape == (B, M, F)
            assert np.array_equal(_f32_bits(got), _f32_bits(_normalize_ref(mid, mean, std))), (F, M, B)


def test_normalize_windows_special_values(C):
    """Zero std (+-inf, and NaN for 0 / 0), NaN and inf in the matrix and the mean, overflow, and subnormal operands and
    results, which must not be flushed to zero."""
    rng = np.random.default_rng(3)
    B, F, M = 3, 40, 70
    tiny = np.finfo(np.float32).tiny
    mid = rng.standard_normal((B, F, M)).astype(np.float32)
    mean = rng.standard_normal(F).astype(np.float32)
    std = rng.uniform(0.5, 2.0, size=F).astype(np.float32)
    std[0] = 0.0                                                        # x / 0: +-inf, and NaN where x == mean
    mid[:, 0, ::3] = mean[0]
    std[1] = -0.0
    mid[0, 2, 5], mid[1, 2, 6], mid[2, 2, 7] = np.nan, np.inf, -np.inf  # non-finite values
    mean[3] = np.inf
    mean[4] = np.nan
    mean[5] = np.float32(3e38)                                          # x - mean overflows where x < -4e37
    mid[:, 5, :] = -np.float32(3e38)
    mid[:, 6, :] = rng.standard_normal((B, M)).astype(np.float32) * np.float32(tiny)           # subnormal operands
    mean[6] = np.float32(3 * tiny / 8)
    std[6] = np.float32(0.7)
    mid[:, 7, :] = rng.standard_normal((B, M)).astype(np.float32) * np.float32(1e-30)          # subnormal quotients
    mean[7] = 0.0
    std[7] = np.float32(3e9)
    mid[:, 8, :] = rng.standard_normal((B, M)).astype(np.float32) * np.float32(1e-40)          # subnormal / subnormal
    mean[8] = 0.0
    std[8] = np.float32(7e-41)
    mid[:, 9, :] = np.float32(2 * tiny)                                 # a subnormal difference of normal values
    mean[9] = np.float32(1.5 * tiny)
    std[9] = 1.0
    with np.errstate(all="ignore"):
        ref = _normalize_ref(mid, mean, std)
    sub = (ref != 0) & (np.abs(ref) < tiny)
    assert sub[..., 6].any() and sub[..., 7].any() and sub[..., 9].all()
    assert np.isnan(ref[..., 0]).any() and np.isinf(ref[..., 0]).any() and np.isinf(ref[..., 5]).all()
    got = _normalize(C, mid, mean, std)
    assert np.array_equal(_f32_bits(got), _f32_bits(ref))


def test_normalize_windows_too_many_clips(C):
    import torch
    from pyaudioanalysis_b200._lib import ERR_UNSUPPORTED, lib
    buf = torch.zeros(16, dtype=torch.float32, device="cuda")
    p = buf.data_ptr()
    assert lib().b200aa_normalize_windows(p, 65536, 2, 2, p, p, p, None) == ERR_UNSUPPORTED
    assert lib().b200aa_normalize_windows(p, 1 << 40, 2, 2, p, p, p, None) == ERR_UNSUPPORTED

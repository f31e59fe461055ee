"""CPU: the last-bit banks of tests/last_bit_cases.py -- permuted kNN pairs, permuted-mean and duplicated-state HMMs, cyclic
cross-validation problems -- against the repository's oracles and the host harnesses (tests/knn_host.cu, hmm_host.cu,
knn_cv_host.cu), bit for bit; every named mutant of the kernels' arithmetic changes a discrete answer on them (the counts
are printed); and a build of tests/knn_host.cu that contracts the distance chain into FMAs changes a classify id."""
import platform

import numpy as np
import pytest
from scipy.spatial.distance import cdist
from sklearn.preprocessing import StandardScaler

from tests import host_exe
from tests import hmm_oracle as H
from tests import knn_cv_oracle
from tests import last_bit_cases as L
from tests.host_exe import bits, floats, hexes, run
from tests.knn_oracle import slots_of

pytestmark = pytest.mark.skipif(host_exe.nvcc() is None, reason="nvcc not available")


@pytest.fixture(scope="module")
def knn_banks():
    return [(b, L.knn_expected(b)) for b in L.knn_banks()]


@pytest.fixture(scope="module")
def hmm_cases():
    return L.hmm_cpu_cases()


@pytest.fixture(scope="module")
def cv_banks():
    return [(bank, knn_cv_oracle.predict(*bank)) for bank in L.cv_banks()]


def _report(capsys, title, rows):
    with capsys.disabled():
        print("\n" + title)
        for name, caught, total, what in rows:
            print("  %-12s %5d of %5d  %s" % (name, caught, total, what))


def _classify(exe, bank):
    slots, C = slots_of(bank.labels)
    N, F = bank.feats.shape
    out = run(exe, "classify %d %d %d %d %s %s %d %s\n" % (N, F, C, bank.k, " ".join(map(str, slots)), hexes(bank.feats),
                                                            bank.queries.shape[0], hexes(bank.queries)))
    return np.array([int(ln[1]) for ln in out]), np.array([floats(ln[2:]) for ln in out])


def _pair_distances(exe, bank):
    """The harness's distances of each query to its own A and B rows, and cdist's."""
    rows = bank.feats[bank.pairs.ravel()]
    out = run(exe, "dist %d %d %d %s %s\n" % (rows.shape[0], bank.F, bank.queries.shape[0], hexes(rows), hexes(bank.queries)))
    n = bank.queries.shape[0]
    sel = (np.arange(n)[:, None], 2 * np.arange(n)[:, None] + np.arange(2)[None, :])
    return np.array([floats(ln[1:]) for ln in out])[sel], cdist(bank.queries, rows)[sel]


# ------------------------------------------------------------------ kNN
@pytest.fixture(scope="module")
def knn_exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "knn_host.cu", "-O1")


def test_knn_banks_are_what_they_claim(knn_banks):
    """Each query's k-th neighbour is the nearer row of its pair under cdist; the pairs sit at every row position of a
    64-row tile, inside one tile and across two, with the lower index on the nearer row and on the farther row; the
    queries fill three 64-query tiles; and there are exact ties, which the lower index decides."""
    positions, same_tile, nearer_low, nearer_high, ties = set(), 0, 0, 0, 0
    for bank, (ids, P) in knn_banks:
        assert all(np.array_equal(a, b) for a, b in zip(L.knn_mutant(bank, "kernel"), (ids, P))), (bank.F, bank.k)
        assert bank.queries.shape[0] > 2 * L.TILE
        d = cdist(bank.queries, bank.feats)
        n = np.arange(bank.queries.shape[0])
        dA, dB = d[n, bank.pairs[:, 0]], d[n, bank.pairs[:, 1]]
        positions |= set((bank.pairs % L.TILE).ravel().tolist())
        same_tile += int((bank.pairs[:, 0] // L.TILE == bank.pairs[:, 1] // L.TILE).sum())
        a_low = bank.pairs[:, 0] < bank.pairs[:, 1]
        nearer_low += int(((dA < dB) & a_low | (dB < dA) & ~a_low).sum())
        nearer_high += int(((dA < dB) & ~a_low | (dB < dA) & a_low).sum())
        ties += int((dA == dB).sum()) if bank.F > 1 else 0
    assert positions == set(range(L.TILE))
    assert same_tile > 0 and nearer_low > 0 and nearer_high > 0 and ties > 0


def test_knn_host_harness_matches_oracle(knn_exe, knn_banks):
    for bank, (ids, P) in knn_banks:
        got = _classify(knn_exe, bank)
        assert np.array_equal(got[0], ids), (bank.F, bank.k)
        assert np.array_equal(got[1], P), (bank.F, bank.k)
        mine, ref = _pair_distances(knn_exe, bank)
        assert np.array_equal(bits(mine), bits(ref)), (bank.F, bank.k)


def test_knn_mutants_are_caught(knn_banks, capsys):
    rows = []
    for name, what in L.KNN_MUTANTS.items():
        caught = total = 0
        for bank, (ids, P) in knn_banks:
            got = L.knn_mutant(bank, name)
            caught += int((~((got[0] == ids) & (got[1] == P).all(axis=1))).sum())
            total += ids.size
        rows.append((name, caught, total, what))
    _report(capsys, "kNN mutants: queries whose (id, P) change", rows)
    assert all(r[1] > 0 for r in rows), rows


def _contract_flags():
    machine = platform.machine().lower()
    if machine in ("x86_64", "amd64"):
        return ("-O2", "-Xcompiler", "-march=haswell,-ffp-contract=fast")
    if machine in ("aarch64", "arm64"):
        return ("-O2", "-Xcompiler", "-ffp-contract=fast")
    pytest.skip("no FMA-contracting host flags known for %s" % machine)


def test_contracted_knn_harness_changes_an_id(tmp_path_factory, knn_banks):
    """The same harness built so that the host compiler may contract (x - v) * (x - v) + s into an FMA: some of its
    distances leave cdist's, and some classify id with them -- what the device code's rounded intrinsics prevent."""
    exe = host_exe.build(tmp_path_factory, "knn_host.cu", *_contract_flags())
    banks = [(b, r) for b, r in knn_banks if b.F >= 136 and b.k == 1]
    moved = sum(int((bits(m) != bits(r)).sum()) for m, r in (_pair_distances(exe, b) for b, _ in banks))
    if moved == 0:
        pytest.skip("the contracted build's distances equal cdist's on the bank: the compiler formed no FMA")
    changed = sum(int((_classify(exe, b)[0] != ids).sum()) for b, (ids, _) in banks)
    assert changed > 0, moved


# ------------------------------------------------------------------ HMM
@pytest.fixture(scope="module")
def hmm_exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "hmm_host.cu", "-O1")


def _clip_feats(case, b, window_major):
    f = np.ascontiguousarray(case.x[b, :, :case.counts[b]], dtype=np.float64)
    return np.ascontiguousarray(f.T).T if window_major else f


def test_hmm_restatement_matches_oracle(hmm_cases):
    """The emissions the kernel adds (in sequence for a feature-major clip of more than one window, else pairwise) are
    hmmlearn's density on the reference's layout, and the paths are the oracle's; the duplicated-state models tie on
    every window of a pair, the permuted ones on some."""
    for case in hmm_cases:
        m = case.model
        var = H.model_logs(m.startprob_, m.transmat_, m.covars_)[2]
        n_ties = 0
        for b in range(len(case.counts)):
            for wm in (False, True):
                feats = _clip_feats(case, b, wm)
                e = L.hmm_emissions(case, b, "kernel", wm)
                assert np.array_equal(bits(e), bits(H.log_density(feats.T, m.means_, var))), (case.C, b, wm)
                path, ties = H.predict(feats, m.startprob_, m.transmat_, m.means_, m.covars_, ties=True)
                assert np.array_equal(L.hmm_mutant(case, b, "kernel", wm), path)
                n_ties += ties
        assert n_ties > 0, (case.C, case.tie)


def test_hmm_host_harness_matches_oracle(hmm_exe, hmm_cases):
    """hmm_host.cu's Viterbi on the oracle's emissions gives the oracle's path; its emissions of the first pair's states
    are the oracle's, bit for bit (pairwise for a one-window clip)."""
    for case in hmm_cases:
        m = case.model
        log_start, log_trans, var = H.model_logs(m.startprob_, m.transmat_, m.covars_)
        konst = case.F * np.log(2 * np.pi) + np.log(var).sum(axis=-1)
        script, want = [], []
        for b, n in enumerate(case.counts):
            e = L.hmm_emissions(case, b)
            script.append("viterbi %d %d %s %s %s\n" % (case.C, n, hexes(log_start), hexes(log_trans), hexes(e)))
        out = run(hmm_exe, "".join(script))
        for b, ln in enumerate(out):
            assert np.array_equal(np.array([int(t) for t in ln[1:]]), L.hmm_expected(case, b)), (case.C, case.tie, b)
        script = []
        for b, n in enumerate(case.counts):
            x = case.x[b, :, :n].T
            for j in L.HMM_PAIRS[case.C][0]:
                script.append("emission %d %d %d %s %s %s %s\n" % (case.F, n, n == 1, float(konst[j]).hex(),
                                                                   hexes(m.means_[j]), hexes(var[j]), hexes(x)))
                want.append(L.hmm_emissions(case, b)[:, j])
        for ln, w in zip(run(hmm_exe, "".join(script)), want):
            assert np.array_equal(bits(floats(ln[1:])), bits(w)), (case.C, case.tie)


def test_hmm_mutants_are_caught(hmm_cases, capsys):
    rows = []
    for name, what in L.HMM_MUTANTS.items():
        caught = total = 0
        for case in hmm_cases:
            for b in range(len(case.counts)):
                for wm in (False, True):
                    caught += int(not np.array_equal(L.hmm_mutant(case, b, name, wm), L.hmm_expected(case, b, wm)))
                    total += 1
        rows.append((name, caught, total, what))
    _report(capsys, "HMM mutants: clip decodes (either layout) whose path changes", rows)
    assert all(r[1] > 0 for r in rows), rows


# ------------------------------------------------------------------ kNN cross-validation
@pytest.fixture(scope="module")
def cv_exe(tmp_path_factory):
    return host_exe.build(tmp_path_factory, "knn_cv_host.cu", "-O1")


def test_cv_banks_are_cyclic_and_match_oracle(cv_banks, cv_exe):
    """Every training matrix, in split order, is cyclic; the splits are not in index order; the restated scaler and
    knn_cv_host.cu's fit are scikit-learn's StandardScaler bit for bit; and the restated predictions are the oracle's."""
    for (X, y, splits, ks), ref in cv_banks:
        for p, ((tr, te), k) in enumerate(zip(splits, ks)):
            Xtr = X[tr]
            n = Xtr.shape[0]
            assert np.array_equal(Xtr, Xtr[0][(np.arange(n)[:, None] + np.arange(n)[None, :]) % n])
            assert not np.array_equal(tr, np.sort(tr))
            sc = StandardScaler().fit(Xtr)
            mean, scale = L.scaler(Xtr)
            assert np.array_equal(bits(mean), bits(sc.mean_)) and np.array_equal(bits(scale), bits(sc.scale_)), p
            out = {t[0]: floats(t[1:]) for t in run(cv_exe, "fit %d %d %d %s %s\n" % (n, len(te), n, hexes(Xtr), hexes(X[te])))}
            assert np.array_equal(bits(out["train"]), bits(sc.transform(Xtr).ravel())), p
            assert np.array_equal(bits(out["test"]), bits(sc.transform(X[te]).ravel())), p
        for a, b in zip(L.cv_predict(X, y, splits, ks), ref):
            assert np.array_equal(a, b)


def test_cv_mutants_are_caught(cv_banks, capsys):
    rows = []
    for name, what in list(L.CV_MUTANTS.items()) + list(L.CV_UNCATCHABLE.items()):
        caught = total = 0
        for bank, ref in cv_banks:
            for a, b in zip(L.cv_predict(*bank, variant=name), ref):
                caught += int(not np.array_equal(a, b))
                total += 1
        rows.append((name, caught, total, what))
    _report(capsys, "kNN cross-validation mutants: problems whose predictions change (the last listed: not catchable)",
            rows)
    for name, caught, _, _ in rows:
        if name in L.CV_UNCATCHABLE:
            assert caught == 0, "%s is caught now: move it to CV_MUTANTS" % name
        else:
            assert caught > 0, name

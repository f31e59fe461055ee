"""Seeded inputs on which one ulp changes a discrete answer, for the kNN (kernel 5), kNN cross-validation (kernel 6) and
HMM decode (kernel 7) kernels, and named mutants: NumPy restatements of each kernel's double arithmetic with one thing
changed, which tests/test_last_bit_cpu.py shows the banks tell apart from the real arithmetic.

Every construction makes two candidates equal in exact arithmetic, so that only the order and rounding of the sums
decides between them:

  kNN      permuted pairs: training rows A and B = A[perm] and a query constant across features.  The two distances add
           the same squared terms in different orders; the label of the nearer row (the lower index on an exact tie)
           decides the vote.
  HMM      permuted means: two states with means a and a[perm], one variance for every feature, uniform transitions,
           and windows holding one value in every feature.  The two log densities add the same terms in different
           orders.  With duplicated states instead (means a and a) every such window is an exact tie, which only the
           Viterbi tie rule decides (csrc/hmm.cuh).
  kNN CV   cyclic training matrices: training row i (in the split's order) is v[(i + f) % n] over F = n features, so
           every column holds the same values and every row is a permutation of every other.  Each column's
           StandardScaler fit adds the same values in another order, and all distances to a constant test row are equal
           in exact arithmetic.
"""
import types
from fractions import Fraction

import numpy as np

from tests import hmm_oracle as H
from tests.knn_oracle import knn_oracle

TILE = 64                                       # rows and queries per tile of knn_dist_kernel
KNN_FEATS = (1, 15, 16, 17, 136, 138)           # one feature, either side of the 16-feature staging step, the real sizes
KNN_KS = (1, 2, 7)
HMM_STATES = (2, 3, 33, 64)
# the states of each model's pairs: lanes j and j + 32 of the Viterbi warp where there are more than 32 states
HMM_PAIRS = {2: [(0, 1)], 3: [(0, 2)], 33: [(0, 32)], 64: [(3, 35), (17, 49), (31, 63)]}


# ------------------------------------------------------------------ sums
def sequential(t):
    """t[..., 0] + t[..., 1] + ... in sequence from +0.0."""
    s = np.zeros(t.shape[:-1])
    for i in range(t.shape[-1]):
        s = s + t[..., i]
    return s


def pairwise(t):
    """NumPy's pairwise summation of the last axis (csrc/npsum.cuh: pairwise_sum)."""
    n = t.shape[-1]
    if n < 8:
        return sequential(t)
    if n <= 128:
        r = [t[..., j] for j in range(8)]
        i = 8
        while i < n - n % 8:
            r = [r[j] + t[..., i + j] for j in range(8)]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(i, n):
            res = res + t[..., i]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise(t[..., :n2]) + pairwise(t[..., n2:])


def restarted(t, step=16):
    """The sum restarted every `step` terms: the blocks' sequential sums added in sequence."""
    return sequential(np.stack([sequential(t[..., a:a + step]) for a in range(0, t.shape[-1], step)], axis=-1))


def reversed_sum(t):
    return sequential(t[..., ::-1])


def fma_chain(d):
    """s = fma(d_i, d_i, s) in sequence from +0.0, each fma rounded once (exact with Fractions): the chain nvcc forms from
    s + d * d when it is allowed to contract.  d: [P, F] -> [P]."""
    out = np.empty(d.shape[0])
    for p, row in enumerate(d):
        s = 0.0
        for x in row.tolist():
            fx = Fraction(x)
            s = float(fx * fx + Fraction(s))
        out[p] = s
    return out


# ------------------------------------------------------------------ kNN (kernel 5)
def knn_bank(seed, F, k, n_q=150, spacing=10.0):
    """Per query p (its value c_p = spacing * p in every feature, exact in float32): a permuted pair A (label 0) and B =
    A[perm] (label 1) with A = c_p + uniform(-1, 1), and k - 1 copies of the query (label 2, distance 0), so that the
    k-th neighbour is the pair's nearer row.  Every other query's rows are at least spacing - 1 per feature further away.
    All rows sit at random indices, so the pairs fall inside and across the 64-row tiles, the lower index on the nearer
    row in some pairs and on the farther row in others; n_q > 128 queries span three 64-query tiles."""
    rng = np.random.default_rng(seed)
    per = k + 1
    N = n_q * per
    c = spacing * np.arange(n_q)
    queries = np.repeat(c[:, None], F, axis=1)
    a = c[:, None] + rng.uniform(-1.0, 1.0, size=(n_q, F))
    b = np.stack([row[rng.permutation(F)] for row in a])
    rows = np.concatenate([a[:, None], b[:, None], np.repeat(queries[:, None], k - 1, axis=1)], axis=1)   # [n_q, per, F]
    labels = np.concatenate([np.zeros((n_q, 1)), np.ones((n_q, 1)), np.full((n_q, k - 1), 2.0)], axis=1)
    where = rng.permutation(N).reshape(n_q, per)                    # the training index of each row
    feats = np.empty((N, F))
    lab = np.empty(N)
    feats[where.ravel()] = rows.reshape(N, F)
    lab[where.ravel()] = labels.ravel()
    return types.SimpleNamespace(F=F, k=k, feats=feats, labels=lab, queries=queries, pairs=where[:, :2].copy())


def knn_banks(seed=500):
    """One bank per (F, k)."""
    return [knn_bank(seed + 10 * i + k, F, k) for i, F in enumerate(KNN_FEATS) for k in KNN_KS]


def chain_terms(bank):
    """(x - v [n_q, F] of each query to its A row, the same to its B row), rounded as the kernel rounds them."""
    d = [bank.queries - bank.feats[bank.pairs[:, s]] for s in (0, 1)]
    return d[0], d[1]


def knn_distances(bank, variant):
    """The squared distances (before sqrt) of each query to its A and its B row under a variant of the chain."""
    dA, dB = chain_terms(bank)
    if variant == "fma":
        return fma_chain(dA), fma_chain(dB)
    f = {"kernel": sequential, "restart16": restarted, "pairwise": pairwise, "reversed": reversed_sum}[variant]
    return f(dA * dA), f(dB * dB)


def knn_outputs(bank, a_wins):
    """(ids, P) of every query when its A row (a_wins) or its B row is the nearer of its pair."""
    k, n_q = bank.k, bank.queries.shape[0]
    C = 2 if k == 1 else 3
    P = np.zeros((n_q, C))
    P[np.arange(n_q), np.where(a_wins, 0, 1)] = 1.0 / k
    if k > 1:
        P[:, 2] = (k - 1) / float(k)
    return np.argmax(P, axis=1), P


def knn_mutant(bank, variant):
    """(ids, P) with the distance chain replaced by `variant`."""
    sA, sB = knn_distances(bank, variant)
    dA, dB = np.sqrt(sA), np.sqrt(sB)
    return knn_outputs(bank, (dA < dB) | ((dA == dB) & (bank.pairs[:, 0] < bank.pairs[:, 1])))


def knn_expected(bank):
    return knn_oracle(bank.feats, bank.labels, bank.k, bank.queries)


KNN_MUTANTS = {
    "fma": "the chain contracted to fma(d, d, s)",
    "restart16": "the chain restarted every 16 features (one per shared-memory stage)",
    "pairwise": "the features summed pairwise instead of in sequence",
    "reversed": "the features added in reverse order",
}


# ------------------------------------------------------------------ HMM (kernel 7)
MEAN_SPREAD, WINDOW_SPREAD = 0.15, 0.05     # of a pair's means and of its windows' values about the pair's centre


def balanced_variance(sq, F):
    """The variance v < sq / F at which F log(2 pi v) + sq / v = 0 (bisection): a window whose squared deviations from
    the means add up to sq then has a log density near 0.  Were the densities near their usual -F / 2 log(2 pi e v),
    K_j would absorb the last bits of the sum, and delta_t, which grows by one density per window, would absorb the
    difference between two states' densities within a few windows."""
    lo, hi = 1e-300, sq / F
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if F * np.log(2 * np.pi * mid) + sq / mid > 0 else (lo, mid)
    return hi


def hmm_model(seed, C, F, tie=False):
    """A C-state diagonal HMM with uniform start and transitions.  Each pair of HMM_PAIRS[C] shares a centre and one
    variance for every feature (balanced_variance of the pair's windows); the second state's means are the first's
    permuted (tie: the same).  The other states sit far from every window."""
    rng = np.random.default_rng(seed)
    means = np.empty((C, F))
    covars = np.empty((C, F))
    paired = set()
    for g, (i, j) in enumerate(HMM_PAIRS[C]):
        dev = MEAN_SPREAD * rng.standard_normal(F)
        a = 6.0 * g + dev
        means[i] = a
        means[j] = a if tie else a[rng.permutation(F)]
        covars[i] = covars[j] = balanced_variance(float((dev * dev).sum()) + F * WINDOW_SPREAD ** 2, F)
        paired |= {i, j}
    for s in range(C):
        if s not in paired:
            means[s] = -40.0 - 3.0 * s + 0.5 * rng.standard_normal(F)
            covars[s] = rng.uniform(0.5, 2.0, size=F)
    return types.SimpleNamespace(startprob_=np.full(C, 1.0 / C), transmat_=np.full((C, C), 1.0 / C), means_=means,
                                 covars_=covars)


def hmm_clips(seed, C, F, counts, M=None, dtype=np.float64):
    """[B, F, M] clips of `dtype` whose window t holds one value in every feature, near the centre of a random pair of
    HMM_PAIRS[C]; NaN past each clip's count, so that a read past it shows."""
    rng = np.random.default_rng(seed)
    M = max(counts) if M is None else M
    centres = 6.0 * np.arange(len(HMM_PAIRS[C]))
    x = np.full((len(counts), F, M), np.nan)
    for b, n in enumerate(counts):
        v = centres[rng.integers(0, centres.size, size=n)] + WINDOW_SPREAD * rng.standard_normal(n)
        x[b, :, :n] = v.astype(dtype)[None, :]
    return x.astype(dtype)


def hmm_case(seed, C, counts, F=136, tie=False, dtype=np.float64, M=None):
    return types.SimpleNamespace(C=C, F=F, tie=tie, counts=list(counts), model=hmm_model(seed, C, F, tie),
                                 x=hmm_clips(seed + 1, C, F, counts, M, dtype))


def hmm_cpu_cases():
    """Per state count: permuted pairs and exact ties, clips of 64 windows and of one window."""
    return [hmm_case(700 + C + 1000 * tie, C, [64] * 10 + [1] * 40, tie=tie) for C in HMM_STATES for tie in (False, True)]


def hmm_expected(case, b, window_major=False):
    """tests/hmm_oracle.py's predict of clip b: features.T (feature-major, the reference's call) or X (window-major)."""
    n = case.counts[b]
    feats = np.ascontiguousarray(case.x[b, :, :n], dtype=np.float64)
    if window_major:
        feats = np.ascontiguousarray(feats.T).T
    m = case.model
    return H.predict(feats, m.startprob_, m.transmat_, m.means_, m.covars_)


def hmm_emissions(case, b, variant="kernel", window_major=False):
    """The log densities [n, C] of clip b as the emission kernel adds them (in sequence over the features for a
    feature-major clip of more than one window, else pairwise), or with one thing changed."""
    n = case.counts[b]
    x = case.x[b, :, :n].astype(np.float64).T                      # [n, F]
    _, _, var = H.model_logs(case.model.startprob_, case.model.transmat_, case.model.covars_)
    mu = case.model.means_
    konst = case.F * np.log(2 * np.pi) + np.log(var).sum(axis=-1)
    d = x[:, None, :] - mu[None, :, :]
    terms = d * d * (1.0 / var) if variant == "recip_var" else d * d / var
    pw = window_major or n == 1
    if variant == "swap_order":
        pw = not pw
    elif variant == "ignore_n1":
        pw = window_major
    if variant == "reversed":
        terms = terms[..., ::-1]
    s = pairwise(terms) if pw else sequential(terms)
    return -0.5 * (konst + s)


def viterbi(log_start, log_trans, frame, first_i=False, last_max=False):
    """hmm_oracle.viterbi with its two tie rules selectable: the backtrack's last i of the maximum (first_i: the first)
    and the first maximum of the final delta (last_max: the last)."""
    n, C = frame.shape
    delta = log_start + frame[0]
    back = np.zeros((n, C), dtype=np.int64)
    for t in range(1, n):
        cand = delta[:, None] + log_trans
        mx = np.fmax.reduce(cand, axis=0, initial=-np.inf)
        back[t] = np.argmax(cand == mx, axis=0) if first_i else C - 1 - np.argmax((cand == mx)[::-1], axis=0)
        delta = mx + frame[t]
    path = np.zeros(n, dtype=np.int64)
    path[-1] = C - 1 - int(np.argmax(delta[::-1])) if last_max else int(np.argmax(delta))
    for t in range(n - 1, 0, -1):
        path[t - 1] = back[t, path[t]]
    return path


def hmm_mutant(case, b, variant, window_major=False):
    """The path of clip b under a mutant of the emission sum or of the Viterbi tie rules."""
    log_start, log_trans, _ = H.model_logs(case.model.startprob_, case.model.transmat_, case.model.covars_)
    e = hmm_emissions(case, b, variant if variant in HMM_EMISSION_MUTANTS else "kernel", window_major)
    return viterbi(log_start, log_trans, e, first_i=variant == "first_i", last_max=variant == "last_max")


HMM_EMISSION_MUTANTS = {
    "swap_order": "pairwise and sequential density sums swapped",
    "reversed": "the density terms added in reverse feature order",
    "recip_var": "(x - mu)^2 multiplied by 1 / var instead of divided by var",
    "ignore_n1": "a one-window feature-major clip summed in sequence (the n == 1 flag ignored)",
}
HMM_MUTANTS = dict(HMM_EMISSION_MUTANTS, first_i="the backtrack takes the first i of the maximum, not the last",
                   last_max="the last state is the last maximum of the final delta, not the first")


# ------------------------------------------------------------------ kNN cross-validation (kernel 6)
def cv_bank(seed, n_problems=8, n=24, m=6, n_classes=3, ks=(1, 1, 3)):
    """(X [R, n], y [R], splits, ks) of n_problems problems on disjoint rows of X at random row indices.  Problem p's
    training rows, in its split's (shuffled) order, form a cyclic matrix v_p[(i + f) % n]; its m test rows hold one
    value each in every feature.  Every class is among each split's training labels."""
    rng = np.random.default_rng(seed)
    R = n_problems * (n + m)
    where = rng.permutation(R).reshape(n_problems, n + m)
    X = np.empty((R, n))
    y = np.empty(R, dtype=np.int64)
    splits = []
    cyc = (np.arange(n)[:, None] + np.arange(n)[None, :]) % n
    for p in range(n_problems):
        tr, te = where[p, :n], where[p, n:]
        v = rng.standard_normal(n) * rng.choice([1e-3, 1.0, 1e3]) + rng.choice([0.0, 5.0, -1e4])
        X[tr] = v[cyc]
        X[te] = (v.mean() + v.std() * rng.standard_normal(m))[:, None]
        y[tr] = rng.permutation(np.arange(n) % n_classes)
        y[te] = rng.integers(0, n_classes, size=m)
        splits.append((tr, te))
    return X, y, splits, [ks[p % len(ks)] for p in range(n_problems)]


def cv_banks():
    return [cv_bank(900 + s) for s in range(8)]


def scaler(Xtr, variant="kernel"):
    """(mean, scale) of StandardScaler().fit(Xtr) as csrc/knn_cv.cuh computes it, rows in Xtr's order, or a mutant."""
    add = {"pairwise": lambda t: pairwise(t.T), "reversed": lambda t: reversed_sum(t.T)}.get(variant, lambda t: sequential(t.T))
    n = Xtr.shape[0]
    s = add(Xtr)
    mean = (0.0 + s) / n
    T = s / n
    c = add(Xtr - T)
    q = add((Xtr - T) ** 2)
    var = q / n if variant == "two_pass" else (q - c * c / n) / n
    eps = np.finfo(np.float64).eps
    drift = n * mean * eps
    constant = var <= n * eps * var + drift * drift
    return mean, np.where(constant, 1.0, np.sqrt(var))


def cv_predict(X, y, splits, ks, variant="kernel"):
    """Per problem the k-NN predictions of its test rows, standardised by a (mutant) scaler fit."""
    out = []
    for (tr, te), k in zip(splits, ks):
        fit_rows = np.sort(tr) if variant == "ascending" else tr
        mean, scale = scaler(X[fit_rows], variant)
        out.append(knn_oracle((X[tr] - mean) / scale, y[tr], int(k), (X[te] - mean) / scale)[0])
    return out


CV_MUTANTS = {
    "pairwise": "the scaler's column sums added pairwise",
    "reversed": "the scaler's column sums added in reverse split order",
    "ascending": "the scaler fitted over the training rows in ascending index order instead of split order",
}
# mutants no bank here can tell apart, and why
CV_UNCATCHABLE = {
    "two_pass": "var = q / n instead of (q - c^2 / n) / n: c, the sum of the deviations from the rounded mean, is so "
                "small on these inputs that c^2 / n does not change q",
}

"""Float64 NumPy restatement of GaussianHMM(C, "diag").predict as the reference calls it (audioSegmentation.py:489,
``hmm.predict(features.T)``): hmmlearn's diagonal log density, evaluated by NumPy on the same array layouts, and its
Viterbi pass, serial in t and vectorised over the states.  Tie rule: the last state is the first maximum of the final
delta; each backtrack step takes the last predecessor of maximal value (DESIGN.md, kernel 7)."""
import numpy as np


def model_logs(start, trans, covars):
    """(log pi, log A, var = max(covars, tiny)) as the host takes them; a zero probability gives -inf."""
    with np.errstate(divide="ignore"):
        return np.log(start), np.log(trans), np.maximum(covars, np.finfo(float).tiny)


def log_density(X, means, var):
    """hmmlearn >= 0.3's _log_multivariate_normal_density_diag of the samples X [n, F] (pass features.T itself: its
    layout decides NumPy's summation order)."""
    nf = means.shape[1]
    return -.5 * (nf * np.log(2 * np.pi) + np.log(var).sum(axis=-1) + ((X[:, None, :] - means) ** 2 / var).sum(axis=-1))


def viterbi(log_start, log_trans, frame, ties=False):
    """The state path [n] of log emission probabilities frame [n, C]; with `ties`, also the number of the path's choices
    (the last state and each backtrack step) that were exact ties, where only the tie rule decided."""
    n, C = frame.shape
    delta = log_start + frame[0]
    back = np.zeros((n, C), dtype=np.int64)
    n_max = np.ones((n, C), dtype=np.int64)
    for t in range(1, n):
        cand = delta[:, None] + log_trans                       # [i, j]
        mx = np.fmax.reduce(cand, axis=0, initial=-np.inf)
        back[t] = C - 1 - np.argmax((cand == mx)[::-1], axis=0)  # the last i of the maximum
        n_max[t] = (cand == mx).sum(axis=0)
        delta = mx + frame[t]
    path = np.zeros(n, dtype=np.int64)
    path[-1] = int(np.argmax(delta))
    for t in range(n - 1, 0, -1):
        path[t - 1] = back[t, path[t]]
    if not ties:
        return path
    return path, int((delta == delta[path[-1]]).sum() > 1) + int((n_max[np.arange(1, n), path[1:]] > 1).sum())


def predict(features, start, trans, means, covars, ties=False, chunk=None):
    """Labels of the windows of features [F, n] (float64), as hmm.predict(features.T) gives them.  `chunk`: evaluate the
    density over that many windows at a time (each chunk laid out as features.T is; chunks of one window would sum
    pairwise, so the last chunk must hold at least two)."""
    log_start, log_trans, var = model_logs(start, trans, covars)
    n = features.shape[1]
    if chunk is None:
        frame = log_density(features.T, means, var)
    else:
        frame = np.concatenate([log_density(np.ascontiguousarray(features[:, a:a + chunk]).T, means, var)
                                for a in range(0, n, chunk)])
    return viterbi(log_start, log_trans, frame, ties)


def path_score(log_start, log_trans, frame, path):
    """The joint log probability of a path, added in the Viterbi recursion's order."""
    s = log_start[path[0]] + frame[0, path[0]]
    for t in range(1, len(path)):
        s = (s + log_trans[path[t - 1], path[t]]) + frame[t, path[t]]
    return s

"""Greedy max-variance data selection restated in numpy, independent of the engine's incremental form.

What the reference's ``GP.update_data`` (gp_class.py:384-471) set out to do, with SURVEY q14 fixed: ``N_new`` times,
append the pool point whose posterior variance summed over the outputs is largest (argmax, ties to the lowest index),
then recompute.  Each step here rebuilds K of the augmented training set, takes a fresh Cholesky factor and evaluates
every pool variance ``sf2_a - |L_a \\ k_a(X, c)|^2`` (noise free, q3) from it: no rank-1 updates, no downdates and no
L^-1, so it shares no algebra with gpmpc_append_greedy beyond the definition.
"""
import numpy as np

from oracle import gp_oracle as orc

try:
    from scipy.linalg import solve_triangular as _solve_tri
except ImportError:  # pragma: no cover
    _solve_tri = None


def pool_variance(X, hyper, Xc):
    """(n, Ny) noise-free posterior variance of every pool point for the training inputs X."""
    X = np.asarray(X, dtype=np.float64); Xc = np.atleast_2d(np.asarray(Xc, dtype=np.float64))
    hyper = np.atleast_2d(np.asarray(hyper, dtype=np.float64))
    Nx = X.shape[1]
    var = np.zeros((Xc.shape[0], hyper.shape[0]))
    for a in range(hyper.shape[0]):
        L = np.linalg.cholesky(orc.assemble_K(X, hyper[a]))
        ks = orc.covSEard(X, Xc, hyper[a, :Nx], hyper[a, Nx] ** 2)
        v = _solve_tri(L, ks, lower=True) if _solve_tri is not None else np.linalg.solve(L, ks)
        var[:, a] = hyper[a, Nx] ** 2 - np.sum(v * v, axis=0)
    return var


def greedy_select(X, hyper, Xc, n_new):
    """Returns dict(picked (n_new,) pool indices in order, score (n_new,) combined variance at pick time,
    gap (n_new,) relative margin of the winner over the runner-up, inf when it was the last candidate)."""
    X = np.asarray(X, dtype=np.float64).copy(); Xc = np.asarray(Xc, dtype=np.float64)
    active = np.ones(Xc.shape[0], dtype=bool)
    picked, score, gap = [], [], []
    for _ in range(int(n_new)):
        var = pool_variance(X, hyper, Xc)
        s = var[:, 0].copy()
        for a in range(1, var.shape[1]):
            s += var[:, a]
        s[~active] = -np.inf
        c = int(np.argmax(s))
        rest = np.delete(s, c)
        second = rest.max() if rest.size and np.isfinite(rest.max()) else -np.inf
        gap.append((s[c] - second) / max(abs(s[c]), 1e-300) if np.isfinite(second) else np.inf)
        picked.append(c); score.append(s[c])
        active[c] = False
        X = np.vstack([X, Xc[c]])
    return dict(picked=np.array(picked, dtype=np.int64), score=np.array(score), gap=np.array(gap))

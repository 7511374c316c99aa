"""The long-double yardstick of the prediction's input derivatives (hess_oracle.predict_derivs_ld, the reference of
test_predict_derivs_shapes_gpu) without a GPU: against a 40-digit mpmath evaluation of the same formulas, against the
float64 closed forms of hess_oracle.predict_hess, and its sums of |terms| against the magnitudes they bound."""
import numpy as np
import pytest
from scipy.linalg import solve_triangular

from oracle import gp_oracle as orc
from oracle import hess_oracle as hor
from tests._util import normalised

OUTS = ('mean', 'var', 'J', 'dvar_dz', 'hess', 'd2var_dz2', 'd3mean_dz3', 'cov', 'dcov_dz', 'd2cov_dz2')
EXTENDED = np.finfo(np.longdouble).eps < 1e-18
needs_ld = pytest.mark.skipif(not EXTENDED, reason='np.longdouble is no wider than float64 here')


def tiny(N=12, Nx=3, Ny=2, H=2, sn=0.3, seed=3):
    """X, hyper, alpha, L^-1 (from the float64 Cholesky factor), chol, Z near training points and a non-symmetric
    per-point Sigma."""
    p = orc.synthetic_problem(N, Nx, Ny, config_id=90 + N, H=H)
    X, Y, hyper = p['X'], p['Y'], p['hyper'].copy()
    hyper[:, Nx + 1] = sn
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    chol = post['chol']
    linv = np.stack([solve_triangular(c, np.eye(N), lower=True) for c in chol])
    rng = np.random.default_rng(seed)
    Z = X[rng.choice(N, H, replace=False)] + 0.1 * rng.standard_normal((H, Nx))
    A = rng.standard_normal((H, Nx, Nx))
    S = 0.05 * (np.eye(Nx) + A @ np.swapaxes(A, 1, 2) / Nx) + 0.02 * (A - np.swapaxes(A, 1, 2))
    return X, hyper, post['alpha'], linv, chol, Z, S


def mp_reference(X, hyper, alpha, linv, Z, S, dps=40):
    """Every output of predict_derivs_ld for 'TA', written out as loops over mpmath numbers at ``dps`` digits."""
    import mpmath as mp
    mp.mp.dps = dps
    f = mp.mpf
    N, Nx = X.shape
    H, Ny = Z.shape[0], hyper.shape[0]
    shapes = dict(mean=(H, Ny), var=(H, Ny), J=(H, Ny, Nx), dvar_dz=(H, Ny, Nx), hess=(H, Ny, Nx, Nx),
                  d2var_dz2=(H, Ny, Nx, Nx), d3mean_dz3=(H, Ny, Nx, Nx, Nx), cov=(H, Ny, Ny), dcov_dz=(H, Ny, Ny, Nx),
                  d2cov_dz2=(H, Ny, Ny, Nx, Nx))
    out = {k: np.zeros(s, dtype=np.longdouble) for k, s in shapes.items()}

    def ld(x):                                      # correctly rounded to long double through a 30-digit string
        return np.longdouble(mp.nstr(x, 30, min_fixed=1, max_fixed=0))
    R = range(Nx)
    for h in range(H):
        Jm, Hm, T3, var, dvar, V2 = [], [], [], [], [], []
        for a in range(Ny):
            ell = [f(hyper[a, d]) for d in R]
            sf2 = f(hyper[a, Nx]) ** 2
            s = [[(f(X[i, d]) - f(Z[h, d])) / ell[d] ** 2 for d in R] for i in range(N)]
            ks = [sf2 * mp.exp(-sum(((f(X[i, d]) - f(Z[h, d])) / ell[d]) ** 2 for d in R) / 2) for i in range(N)]
            Li = [[f(linv[a, i, j]) for j in range(N)] for i in range(N)]
            v = [mp.fsum(Li[i][j] * ks[j] for j in range(N)) for i in range(N)]
            beta = [mp.fsum(Li[j][i] * v[j] for j in range(N)) for i in range(N)]
            Vd = [[mp.fsum(Li[i][j] * ks[j] * s[j][d] for j in range(N)) for i in range(N)] for d in R]
            wa = [f(alpha[a, i]) * ks[i] for i in range(N)]
            wb = [beta[i] * ks[i] for i in range(N)]
            mean = mp.fsum(wa)
            q = mp.fsum(x * x for x in v)
            J = [mp.fsum(wa[i] * s[i][d] for i in range(N)) for d in R]
            Hd = [[mp.fsum(wa[i] * s[i][d] * s[i][e] for i in range(N)) - (mean / ell[d] ** 2 if d == e else 0)
                   for e in R] for d in R]
            dv = [-2 * mp.fsum(wb[i] * s[i][d] for i in range(N)) for d in R]
            v2 = [[-2 * (mp.fsum(Vd[d][i] * Vd[e][i] for i in range(N)) + mp.fsum(wb[i] * s[i][d] * s[i][e] for i in range(N))
                         - (q / ell[d] ** 2 if d == e else 0)) for e in R] for d in R]
            t3 = [[[mp.fsum(wa[i] * s[i][d] * s[i][e] * s[i][g] for i in range(N))
                    - (J[g] / ell[d] ** 2 if d == e else 0) - (J[e] / ell[d] ** 2 if d == g else 0)
                    - (J[d] / ell[e] ** 2 if e == g else 0) for g in R] for e in R] for d in R]
            Jm.append(J); Hm.append(Hd); T3.append(t3); var.append(sf2 - q); dvar.append(dv); V2.append(v2)
            out['mean'][h, a] = ld(mean); out['var'][h, a] = ld(sf2 - q)
            out['J'][h, a] = [ld(x) for x in J]; out['dvar_dz'][h, a] = [ld(x) for x in dv]
            out['hess'][h, a] = [[ld(x) for x in r] for r in Hd]
            out['d2var_dz2'][h, a] = [[ld(x) for x in r] for r in v2]
            out['d3mean_dz3'][h, a] = [[[ld(x) for x in r] for r in p] for p in t3]
        Sg = [[f(S[h, d, e]) for e in R] for d in R]
        for a in range(Ny):
            for b in range(Ny):
                dab = 1 if a == b else 0
                out['cov'][h, a, b] = ld(dab * var[a] + mp.fsum(Jm[a][d] * Sg[d][e] * Jm[b][e] for d in R for e in R))
                for g in R:
                    out['dcov_dz'][h, a, b, g] = ld(dab * dvar[a][g] + mp.fsum(
                        Hm[a][d][g] * Sg[d][e] * Jm[b][e] + Jm[a][d] * Sg[d][e] * Hm[b][e][g] for d in R for e in R))
                    for k in R:
                        out['d2cov_dz2'][h, a, b, g, k] = ld(dab * V2[a][g][k] + mp.fsum(
                            T3[a][d][g][k] * Sg[d][e] * Jm[b][e] + Hm[a][d][g] * Sg[d][e] * Hm[b][e][k]
                            + Hm[a][d][k] * Sg[d][e] * Hm[b][e][g] + Jm[a][d] * Sg[d][e] * T3[b][e][g][k]
                            for d in R for e in R))
    return out


@needs_ld
def test_long_double_reference_vs_mpmath():
    """N = 12, Nx = 3, Ny = 2, H = 2, TA with a non-symmetric per-point Sigma: every output within 1e-17 of the 40-digit
    evaluation, normalised by its sum of |terms| (long double's unit roundoff is 5.4e-20)."""
    pytest.importorskip('mpmath')
    X, hyper, alpha, linv, _, Z, S = tiny()
    ref = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, 'TA')
    ab = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, 'TA', absolute=True)
    mp = mp_reference(X, hyper, alpha, linv, Z, S)
    errs = {k: normalised(ref[k], mp[k], ab[k]) for k in OUTS}
    assert max(errs.values()) <= 1e-17, errs


@pytest.mark.parametrize('method', ['TA', 'ME'])
def test_long_double_reference_vs_float64_closed_forms(method):
    """At sn = 0.3 with L^-1 = inv(chol) the long-double path and predict_hess's triangular solves agree to 1e-12 of the
    sums of |terms| (the two differ by how K^-1 is applied, not by the formulas)."""
    X, hyper, alpha, linv, chol, Z, S = tiny(N=60, Nx=4, Ny=3, H=3)
    ref = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, method)
    ab = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, method, absolute=True)
    cf = hor.predict_hess(X, hyper, alpha, chol, Z, S if method == 'TA' else None, method)
    pairs = dict(mean='mean', var='var', J='dmean', dvar_dz='dvar', hess='hess', d2var_dz2='d2var', d3mean_dz3='d3mean',
                 dcov_dz='dcov', d2cov_dz2='d2cov')
    errs = {k: normalised(cf[c], ref[k], ab[k]) for k, c in pairs.items()}
    assert max(errs.values()) <= 1e-12, errs


def test_absolute_sums_bound_the_results():
    """Every sum of |terms| is at least the magnitude of the result it normalises, and strictly positive where the
    result is not zero."""
    X, hyper, alpha, linv, _, Z, S = tiny(N=60, Nx=4, Ny=3, H=3)
    for method, Sg in (('TA', S), ('TA', S[0]), ('ME', None)):
        ref = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, Sg, method)
        ab = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, Sg, method, absolute=True)
        for k in OUTS:
            assert ref[k].dtype == np.longdouble and ref[k].shape == ab[k].shape, k
            assert np.all(ab[k] >= np.abs(ref[k])), (method, k)

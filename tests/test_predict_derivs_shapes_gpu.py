"""The prediction's input derivatives (gpmpc_predict_hess; its first seven outputs are gpmpc_predict_grad's bit for bit)
against the long-double restatement hess_oracle.predict_derivs_ld fed the engine's own alpha and L^-1, at every shape the
derivative kernels branch on:

* the register extent NXP of grad_reduce / hess_reduce (8 / 16 / 32: Nx = 1, 8, 9, 16, 17, 24, 32), with their pair
  rounds (Nx = 24: 300 pairs, Nx = 32: 528, the third round) and triple rounds (Nx = 16: 4, Nx = 24: 11, Nx = 32: all 24);
* R = 64 / Nx points per derivative pass (64, 8, 7, 4, 3, 2 and a partial last pass), so the derivative product runs at
  BM 64 and BM 16, and at Nx = 9 over rows of dDR a longer pass left behind;
* 1024-point GR_CHUNK blocks: one, two with a 6-point last block (N = 1030), three (N = 2150), and odd tile counts of
  Npad (1152, 2176) where the upper-mode beta product ends in a half tile;
* 64-point chunks of H (65 and 130 points: a last chunk of one and of two points), Ny = 1 and Ny = 9;
* a reserved handle (Npad 2176 for N = 1900), whose L^-1 and U = L^-T have an identity tail inside both products;
* TA with one shared Sigma, a per-point stack and a non-symmetric Sigma, and ME.

Errors are normalised entry by entry by the sum of |terms| of each output (predict_derivs_ld(..., absolute=True)), which
follows the cancellation inside L^-1 ks as well as the one in each sum; cond(K) enters neither side, since the reference
takes the engine's alpha and L^-1.  Before any comparison the guards require every term a kernel could lose -- each
live 1024-point block of each output, the Sigma terms of dcov / d2cov, the transposition of a non-symmetric Sigma -- to
move some entry by at least 1e4 x the bar x its normaliser.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, largest normalised error over every case, ME and the three
TA ways (case in brackets):

    mean 5.7e-17 (ny1)   var 1.7e-18 (nx32)   cov 6.4e-18 (nx1)     jac 8.8e-17 (ny1)         dvar_dz 2.0e-18 (nx24)
    dcov_dz 3.1e-18 (nx1)   hess 3.3e-16 (nx17)   d2var_dz2 4.2e-18 (nx24)   d3mean_dz3 6.4e-16 (ny9)   d2cov_dz2 4.2e-18 (nx24)

and at sn = 1e-2 (nx8, cond(K) ~ 1e7) no larger: mean 2.0e-17, jac 3.3e-17, hess 1.2e-16, d3mean_dz3 1.5e-16, the rest
<= 1.4e-20.  The outputs built from alpha ks alone (mean, jac, hess, d3mean_dz3) carry the few-ulp error of each ks; the
ones through L^-1 are normalised by sums that include |L^-1| ks, so their errors are orders of magnitude smaller.
PREDICT_TOL (tests/_util.py) is 10x each maximum rounded up to a power of ten.  The smallest guard ratios, all at
sn = 1e-2, are 3.0e-10 (a block of d2var_dz2) and 5.7e-10 (dvar_dz), 4.1e-8 (the Sigma terms of dcov_dz) and 1.1e-8 (Sigma^T in dcov_dz), against the
guard's 1e4 x 1e-16; a block of hess or d3mean_dz3 moves them by >= 3.9e-3 against 1e4 x 1e-14."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import hess_oracle as hor
from oracle import gp_oracle as orc
from tests._util import PREDICT_TOL, normalised

pytestmark = pytest.mark.gpu

# name -> (N, Nx, Ny, H, capacity or None, sn)
CASES = {
    'nx1': (200, 1, 2, 65, None, 0.3),           # NXP 8, one live dimension; R = 64 (BM 64), chunks of 64 and 1 point
    'nx8': (1030, 8, 3, 9, None, 0.3),           # top of the 8 bucket; blocks of 1024 and 6; passes of 8 and 1; Npad 1152
    'nx8_sn1e-2': (1030, 8, 3, 9, None, 1e-2),   # the same with cond(K) ~ 1e7
    'nx9': (700, 9, 2, 8, None, 0.3),            # bottom of the 16 bucket; R = 7: 63 rows at BM 64, then 9 at BM 16
    'nx16': (2150, 16, 2, 5, None, 0.3),         # top of the 16 bucket, all 4 triple rounds; three blocks; Npad 2176
    'nx17': (300, 17, 2, 4, None, 0.3),          # NXP 32, R = 3
    'nx24': (500, 24, 2, 3, None, 0.3),          # second pair round (300 pairs), 11 triple rounds
    'nx32': (1100, 32, 2, 3, None, 0.3),         # third pair round (528 pairs), 24 triple rounds; R = 2; two blocks
    'ny1': (129, 5, 1, 64, None, 0.3),           # one output; Npad 256; one full 64-point chunk
    'ny9': (400, 4, 9, 130, None, 0.3),          # Ny > 8; chunks of 64, 64 and 2 points
    'reserved': (1900, 6, 2, 9, 2100, 0.3),      # Npad 2176 instead of 1920: identity tails of L^-1 and U
}
FAMILIES = ('mean', 'var', 'cov', 'jac', 'dvar_dz', 'dcov_dz', 'hess', 'd2var_dz2', 'd3mean_dz3', 'd2cov_dz2')
REF_KEY = dict(jac='J')
GUARD = 1e4
# the three TA ways: one shared Sigma (spp 0), a per-point stack (spp 1), a non-symmetric shared Sigma
SIGMA_WAYS = ('shared', 'stack', 'skew')


def problem(name, H=None, seed=0):
    """X, Y, hyper (sn of the case) and H test points 0.05 away from training points spread evenly over [0, N), so every
    1024-point block, the last partial one included, has test points near its data."""
    N, Nx, Ny, Hc, _, sn = CASES[name]
    H = Hc if H is None else H
    p = orc.synthetic_problem(N, Nx, Ny, config_id=600 + Nx + Ny, H=1)
    hyper = p['hyper'].copy()
    hyper[:, Nx + 1] = sn
    idx = np.round(np.linspace(0, N - 1, H)).astype(int)
    Z = p['X'][idx] + 0.05 * np.random.default_rng(seed + Nx).standard_normal((H, Nx))
    return p['X'], p['Y'], hyper, Z


def sigmas(hyper, H):
    """{'shared': 0.1 Lambda^1/2 (I + C) Lambda^1/2 / 2 with C a random correlation matrix and Lambda = diag(ell^2) of the
    output with the smallest length scales, 'stack': (H,Nx,Nx) of it scaled by 1 + 0.05 h, 'skew': it plus a
    skew-symmetric part of 0.3 x its size}."""
    Nx = hyper.shape[1] - 2
    ell = hyper[np.argmin(np.sum(np.log(hyper[:, :Nx]), 1)), :Nx]
    rng = np.random.default_rng(70 + Nx)
    A = rng.standard_normal((Nx, Nx))
    M = A @ A.T
    d = np.sqrt(np.diag(M))
    S = 0.1 * ell[:, None] * (0.5 * (np.eye(Nx) + M / np.outer(d, d))) * ell[None, :]
    B = rng.standard_normal((Nx, Nx))
    K = B - B.T
    skew = S + (0.3 * np.linalg.norm(S) / np.linalg.norm(K) * K if Nx > 1 else 0.0)
    stack = np.stack([S * (1 + 0.05 * h) for h in range(H)])
    return dict(shared=S, stack=stack, skew=skew)


def fit(name):
    import gp_mpc_b200
    N, Nx, Ny, _, cap, _ = CASES[name]
    X, Y, hyper, Z = problem(name)
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0, capacity=cap)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)
    assert not eng.factorize().any()
    return eng, X, Y, hyper, Z


def engine_factor(eng, Ny):
    """The engine's alpha (Ny, N) and L^-1 (Ny, N, N)."""
    return (np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)]),
            np.stack([eng.get(L.GET_LINV, a) for a in range(Ny)]))


def block_terms(X, hyper, alpha, linv, Z, lo, hi):
    """What leaving the training points [lo, hi) out of the reductions removes from dvar_dz, hess, d2var_dz2 and
    d3mean_dz3 (float64; a dropped GR_CHUNK block of grad_reduce / hess_reduce / their finalize loses exactly this)."""
    Nx = X.shape[1]
    H, Ny = Z.shape[0], hyper.shape[0]
    out = dict(dvar_dz=np.zeros((H, Ny, Nx)), hess=np.zeros((H, Ny, Nx, Nx)), d2var_dz2=np.zeros((H, Ny, Nx, Nx)),
               d3mean_dz3=np.zeros((H, Ny, Nx, Nx, Nx)))
    for a in range(Ny):
        ell = hyper[a, :Nx]
        ks = orc.covSEard(X, Z, ell, hyper[a, Nx] ** 2).T              # (H,N)
        s = (X[None] - Z[:, None]) / ell ** 2                          # (H,N,Nx)
        beta = linv[a].T @ (linv[a] @ ks.T)                            # (N,H)
        Vd = np.einsum('ij,hjd->ihd', linv[a], ks[:, :, None] * s)     # (N,H,Nx)
        wa, wb, sb, Vb = (alpha[a] * ks)[:, lo:hi], (beta.T * ks)[:, lo:hi], s[:, lo:hi], Vd[lo:hi]
        out['dvar_dz'][:, a] = -2 * np.einsum('hi,hid->hd', wb, sb)
        out['hess'][:, a] = np.einsum('hi,hid,hie->hde', wa, sb, sb)
        out['d2var_dz2'][:, a] = -2 * (np.einsum('ihd,ihe->hde', Vb, Vb) + np.einsum('hi,hid,hie->hde', wb, sb, sb))
        out['d3mean_dz3'][:, a] = np.einsum('hi,hid,hie,hif->hdef', wa, sb, sb, sb, optimize=True)
    return out


def guard_ratio(part, scale):
    """The largest |part| / scale: how far above the normaliser a term a kernel could drop stands."""
    return float(np.max(np.abs(part) / np.where(scale > 0, scale, np.inf)))


def check_guards(X, hyper, alpha, linv, Z, core, core_abs, S):
    """Every live block of every output, and (given TA Sigmas) the Sigma terms and the transposition of the skew Sigma,
    move some entry of their outputs by >= GUARD x the bar x the normaliser.  Returns the smallest ratio seen per guard."""
    N = X.shape[0]
    Ny = hyper.shape[0]
    seen = {}
    for lo in range(0, N, 1024):
        part = block_terms(X, hyper, alpha, linv, Z, lo, min(N, lo + 1024))
        for k, v in part.items():
            for a in range(Ny):
                r = guard_ratio(v[:, a], core_abs[k][:, a])
                assert r >= GUARD * PREDICT_TOL[k], ('block', lo, a, k, r)
                seen['block ' + k] = min(seen.get('block ' + k, np.inf), r)
    if S is not None:
        me = hor.cov_derivs(core, None, 'ME')
        for way in SIGMA_WAYS:
            ta = hor.cov_derivs(core, S[way], 'TA')
            ab = hor.cov_derivs(core_abs, np.abs(S[way]), 'TA')
            for k in ('dcov_dz', 'd2cov_dz2'):
                r = guard_ratio(ta[k] - me[k], ab[k])
                assert r >= GUARD * PREDICT_TOL[k], ('Sigma terms', way, k, r)
                seen['Sigma ' + k] = min(seen.get('Sigma ' + k, np.inf), r)
    # Sigma -> Sigma^T leaves the a = b blocks unchanged (Hm_a and T_a are symmetric in their derivative indices), so
    # only a pair of outputs, and only Nx > 1, can tell a transposed Sigma apart
    if S is not None and X.shape[1] > 1 and hyper.shape[0] > 1:
        tr = hor.cov_derivs(core, S['skew'].T, 'TA')
        sk = hor.cov_derivs(core, S['skew'], 'TA')
        ab = hor.cov_derivs(core_abs, np.abs(S['skew']), 'TA')
        for k in ('dcov_dz', 'd2cov_dz2'):
            r = guard_ratio(tr[k] - sk[k], ab[k])
            assert r >= GUARD * PREDICT_TOL[k], ('Sigma^T', k, r)
            seen['Sigma^T ' + k] = r
    return seen


def case_errors(name):
    """Per call ('ME', 'TA shared', 'TA stack', 'TA skew'): the largest normalised error of each output family, after
    the guards (their smallest ratios under 'guards').  On the reserved handle every call is repeated and must give the
    same bits."""
    _, Nx, Ny, H, _, _ = CASES[name]
    eng, X, Y, hyper, Z = fit(name)
    alpha, linv = engine_factor(eng, Ny)
    S = sigmas(hyper, H)
    calls = {'ME': (L.METHOD_ME, None, 'ME')}
    calls.update({'TA ' + w: (L.METHOD_TA, S[w], 'TA') for w in SIGMA_WAYS})
    outs = {c: eng.predict_hess(Z, Sg, m) for c, (m, Sg, _) in calls.items()}
    if name == 'reserved':
        for c, (m, Sg, _) in calls.items():
            again = eng.predict_hess(Z, Sg, m)
            for k in FAMILIES:
                assert np.array_equal(outs[c][k], again[k]), (c, k)
    eng.close()
    core = hor.derivs_core_ld(X, hyper, alpha, linv, Z)
    core_abs = hor.derivs_core_ld(X, hyper, alpha, linv, Z, absolute=True)
    res = dict(guards=check_guards(X, hyper, alpha, linv, Z, core, core_abs, S))
    for c, (_, Sg, meth) in calls.items():
        ref = dict(core, **hor.cov_derivs(core, Sg, meth))
        ab = dict(core_abs, **hor.cov_derivs(core_abs, None if Sg is None else np.abs(Sg), meth))
        res[c] = {k: normalised(outs[c][k], ref[REF_KEY.get(k, k)], ab[REF_KEY.get(k, k)]) for k in FAMILIES}
    return res


@pytest.mark.parametrize('name', list(CASES))
def test_predict_derivs_vs_long_double(name):
    """Every output of ME and of the three TA ways against the reference, within PREDICT_TOL of the sums of |terms|,
    after the guards."""
    res = case_errors(name)
    for c, errs in res.items():
        if c == 'guards':
            continue
        bad = {k: e for k, e in errs.items() if not e <= PREDICT_TOL[k]}
        assert not bad, (name, c, bad)


@pytest.mark.parametrize('name', ['nx9', 'ny9'])
def test_derivs_do_not_depend_on_batch_or_row(name):
    """A point's outputs have the same bits in batches of 1, R, R + 1, 64 and 65 points at permuted rows, for ME and for
    TA with a per-point Sigma: every sum of the derivative chain runs in a fixed order whatever the batch, and the
    derivative product gives a row the same bits at BM 64 and BM 16."""
    _, Nx, Ny, _, _, _ = CASES[name]
    R = 64 // Nx
    eng, X, Y, hyper, _ = fit(name)
    _, _, _, Z = problem(name, H=65, seed=1)
    S = sigmas(hyper, 65)['stack']
    rng = np.random.default_rng(11)
    for m, Sg in ((L.METHOD_ME, None), (L.METHOD_TA, S)):
        base = eng.predict_hess(Z, Sg, m)
        for H in (1, R, R + 1, 64, 65):
            rows = rng.permutation(65)[:H]
            o = eng.predict_hess(Z[rows], None if Sg is None else Sg[rows], m)
            for k in FAMILIES:
                assert np.array_equal(o[k], base[k][rows]), (m, H, k)
    eng.close()

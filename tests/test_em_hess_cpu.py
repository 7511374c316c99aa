"""Second derivatives of 'EM' exact moment matching without a GPU: the closed-form oracle against fourth-order differences
of the first-derivative oracle in z and along symmetric Sigma perturbations, the heat-equation identities and the index
symmetries inside it, its limit at Sigma = 0 against the ME / TA Hessian oracle, the C declarations, and
GP.predict_batch_em_hess's chain rule through the scalers (on an engine stand-in made of the oracles)."""
import os
import re

import numpy as np
import pytest
from scipy.linalg import cho_solve

import gp_mpc_b200
from oracle import em_grad_oracle as emg
from oracle import em_hess_oracle as emh
from oracle import gp_oracle as orc
from oracle import hess_oracle as hor
from tests._fake_engine import OracleEngine
from tests._util import d4, load_fixture, relinf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _problem(case):
    if case in ('tank', 'car'):
        m = load_fixture(case); X, Y, hyper = m['X'], m['Y'], m['hyper']
        rng = np.random.default_rng(5)
        Z = X[:1] + 0.05 * rng.standard_normal((1, X.shape[1]))
        A = rng.standard_normal((X.shape[1],) * 2); Sigma = 1e-3 * np.eye(X.shape[1]) + 1e-4 * A @ A.T
    else:
        p = orc.synthetic_problem(120, 4, 2, config_id=31, H=1)
        X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'].copy(), p['Z'], p['Sigma']
        hyper[:, X.shape[1] + 1] = 0.3
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    chol = post['chol']
    alpha = np.stack([cho_solve((chol[a], True), Y[:, a]) for a in range(Y.shape[1])])
    return X, Y, hyper, Z, Sigma, alpha, chol


@pytest.mark.parametrize('case', ['tank', 'car', 'syn'])
def test_em_hess_oracle_vs_differences_of_the_gradient_oracle(case):
    X, Y, hyper, Z, Sigma, alpha, chol = _problem(case)
    Nx = X.shape[1]
    cl = emh.em_hess_closed(X, hyper, alpha, chol, Z, Sigma)
    g = lambda z, S: emg.em_grad_closed(X, hyper, alpha, chol, z, S)
    tol = 1e-4 if case == 'car' else 1e-6
    tc = 1e-3 if case == 'car' else 2e-5         # the gradient oracle's cov derivatives are differences of O(1) sums
    fz = {k: np.zeros_like(cl[k2]) for k, k2 in (('dmean_dz', 'd2mean_dz2'), ('dmean_dSigma', 'd2mean_dSigma_dz'),
                                                 ('dcov_dz', 'd2cov_dz2'), ('dcov_dSigma', 'd2cov_dSigma_dz'))}
    for f in range(Nx):
        e = np.zeros(Nx); e[f] = 1.0
        d = d4(lambda s: g(Z + s * e, Sigma), 1e-2)
        for k in fz:
            fz[k][..., f] = d[k]
    assert relinf(cl['d2mean_dz2'], fz['dmean_dz']) < tol
    assert relinf(cl['d2mean_dSigma_dz'], fz['dmean_dSigma']) < tol
    assert relinf(cl['d2cov_dz2'], fz['dcov_dz']) < tc
    assert relinf(cl['d2cov_dSigma_dz'], fz['dcov_dSigma']) < tc
    for f in range(Nx):
        for gg in range(f + 1):
            E = np.zeros((Nx, Nx)); E[f, gg] = E[gg, f] = 1.0
            d = d4(lambda s: g(Z, Sigma + s * E), 1e-4)
            scale = 1.0 if f == gg else 2.0
            assert relinf(scale * cl['d2mean_dSigma2'][..., f, gg], d['dmean_dSigma']) < tol, (f, gg)
            if case != 'car':       # car's cond(K) ~ 1e10 noise in the gradient oracle's cov, amplified by 1 / 1e-4
                assert relinf(scale * cl['d2cov_dSigma2'][..., f, gg], d['dcov_dSigma']) < tc, (f, gg)


def test_em_hess_oracle_identities_and_symmetries():
    X, Y, hyper, Z, Sigma, alpha, chol = _problem('syn')
    cl = emh.em_hess_closed(X, hyper, alpha, chol, Z, Sigma)
    gr = emg.em_grad_closed(X, hyper, alpha, chol, Z, Sigma)
    # heat equation: d mean/dSigma = 1/2 d^2 mean/dz^2, d cov/dSigma = 1/2 d^2 cov/dz^2 + sym(J_a J_b^T)
    assert relinf(gr['dmean_dSigma'], 0.5 * cl['d2mean_dz2']) < 1e-12
    J = gr['dmean_dz']
    JJ = np.einsum('had,hbe->habde', J, J)
    assert relinf(gr['dcov_dSigma'], 0.5 * cl['d2cov_dz2'] + 0.5 * (JJ + np.swapaxes(JJ, 1, 2))) < 1e-10
    assert relinf(cl['d2mean_dSigma_dz'], 0.5 * cl['d3mean_dz3']) == 0
    m4 = cl['d2mean_dSigma2']
    for perm in ((0, 1, 3, 2, 4, 5), (0, 1, 2, 4, 3, 5), (0, 1, 2, 5, 4, 3), (0, 1, 4, 5, 2, 3)):
        assert relinf(np.transpose(m4, perm), m4) < 1e-12
    c4 = cl['d2cov_dSigma2']
    for perm in ((0, 2, 1, 3, 4, 5, 6), (0, 1, 2, 4, 3, 5, 6), (0, 1, 2, 3, 4, 6, 5), (0, 1, 2, 5, 6, 3, 4)):
        assert relinf(np.transpose(c4, perm), c4) < 1e-10
    c3 = cl['d2cov_dSigma_dz']
    assert relinf(np.swapaxes(c3, 3, 4), c3) < 1e-12 and relinf(np.swapaxes(c3, 1, 2), c3) < 1e-12


def test_em_hess_oracle_at_zero_sigma_against_the_me_ta_hessian():
    """Sigma = 0: d2mean_dz2 is the ME mean Hessian, d2mean_dSigma_dz half its third derivative, the diagonal of d2cov_dz2
    the Hessian of var and its off-diagonal zero, and d2cov_dSigma_dz for a != b the symmetrised TA mixed term."""
    X, Y, hyper, Z, _, alpha, chol = _problem('tank')
    Nx, Ny = X.shape[1], Y.shape[1]
    S = np.zeros((Nx, Nx))
    cl = emh.em_hess_closed(X, hyper, alpha, chol, Z, S)
    me = hor.predict_hess(X, hyper, alpha, chol, Z, None, 'ME')
    assert relinf(cl['d2mean_dz2'], me['hess']) < 1e-10
    assert relinf(cl['d2mean_dSigma_dz'], 0.5 * me['d3mean']) < 1e-10
    for a in range(Ny):
        assert relinf(cl['d2cov_dz2'][:, a, a], me['d2var'][:, a]) < 1e-7
        for b in range(Ny):
            J, Hm = me['dmean'], me['hess']
            if a != b:
                assert np.abs(cl['d2cov_dz2'][:, a, b]).max() < 1e-7 * np.abs(me['d2var']).max()
                mix = np.einsum('hdf,he->hdef', Hm[:, a], J[:, b]) + np.einsum('hd,hef->hdef', J[:, a], Hm[:, b])
                ta = 0.5 * (mix + np.swapaxes(mix, 1, 2))
                assert relinf(cl['d2cov_dSigma_dz'][:, a, b], ta) < 1e-7


def test_header_declares_em_hess():
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    m = re.search(r'int gpmpc_predict_em_hess\(([^;]*)\);', hdr)
    assert m and m.group(1).count('double*') == 15
    cas = open(os.path.join(ROOT, 'include', 'gpmpc_casadi.h')).read()
    assert re.search(r'int gp_b200_bind_em_hess\(gpmpc_handle_t h, int Nt\);', cas)


class _EmEngine(OracleEngine):
    def predict_em_grad(self, Z, Sigma):
        return emg.em_grad_closed(self.X, self.hyper, self.post['alpha'], self.post['chol'], Z, Sigma)

    def predict_em_hess(self, Z, Sigma):
        out = self.predict_em_grad(Z, Sigma)
        h = emh.em_hess_closed(self.X, self.hyper, self.post['alpha'], self.post['chol'], Z, Sigma)
        out.update({k: h[k] for k in emh.KEYS})
        return out


def test_gp_predict_batch_em_hess_chain_rule():
    """Against fourth-order differences of predict_batch_grad(method='EM') in the caller's units: a wrong scale factor
    is off by stdY or stdZ (O(1)), the differences by about 1e-5."""
    m = load_fixture('tank')
    assert m['normalize']
    gp = gp_mpc_b200.GP(m['X'], m['Y'], mean_func='zero', gp_method='EM', normalize=True, hyper=dict(hyper=m['hyper']),
                        engine_factory=_EmEngine, meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    Ny, Nx = m['Y'].shape[1], m['X'].shape[1]
    rng = np.random.default_rng(2)
    x = np.asarray(m['xlb']) + (np.asarray(m['xub']) - np.asarray(m['xlb'])) * rng.random((1, Ny))
    u = np.asarray(m['ulb']) + (np.asarray(m['uub']) - np.asarray(m['ulb'])) * rng.random((1, Nx - Ny))
    S = 1e-3 * np.eye(Nx)
    h = gp.predict_batch_em_hess(x, u, S)
    g = gp.predict_batch_grad(x, u, S, method='EM')
    for k in g:
        assert np.array_equal(h[k], g[k]), k
    z = np.hstack([x, u])
    for f in range(Nx):
        st = 1e-3 * max(1.0, abs(z[0, f]))
        e = np.zeros(Nx); e[f] = st
        d = d4(lambda s: gp.predict_batch_grad((z + s * e / st)[:, :Ny], (z + s * e / st)[:, Ny:], S, method='EM'), st)
        assert relinf(h['d2mean_dz2'][..., f], d['dmean_dz']) < 1e-4
        assert relinf(h['d2mean_dSigma_dz'][..., f], d['dmean_dSigma']) < 1e-4
        assert relinf(h['d2cov_dz2'][..., f], d['dcov_dz']) < 1e-3
        assert relinf(h['d2cov_dSigma_dz'][..., f], d['dcov_dSigma']) < 1e-3
    E = np.zeros((Nx, Nx)); E[0, 1] = E[1, 0] = 1.0
    d = d4(lambda s: gp.predict_batch_grad(x, u, S + s * E, method='EM'), 1e-4)
    assert relinf(2 * h['d2mean_dSigma2'][..., 0, 1], d['dmean_dSigma']) < 1e-4
    assert relinf(2 * h['d2cov_dSigma2'][..., 0, 1], d['dcov_dSigma']) < 1e-3

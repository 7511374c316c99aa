"""First derivatives of 'EM' exact moment matching without a GPU: the closed-form oracle against fourth-order
differences of the extended-precision EM formula, its limits as Sigma -> 0, and its mean and cov against the
extended-precision formula at large input covariances."""
import numpy as np
import pytest
from scipy.linalg import cho_solve

from oracle import em_grad_oracle as emo
from oracle import gp_oracle as orc
from oracle import hess_oracle as hor
from tests._em_cases import sigmas
from tests._util import load_fixture, relinf


def _problem(case):
    if case == 'tank':
        m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
        rng = np.random.default_rng(5)
        Z = X[:2] + 0.05 * rng.standard_normal((2, X.shape[1]))
        A = rng.standard_normal((X.shape[1],) * 2); Sigma = 1e-3 * np.eye(X.shape[1]) + 1e-4 * A @ A.T
    else:
        p = orc.synthetic_problem(300, 6, 3, config_id=21, H=2)
        X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'], p['Sigma']
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    chol = post['chol']
    invK = np.stack([cho_solve((chol[a], True), np.eye(X.shape[0])) for a in range(Y.shape[1])])
    alpha = np.stack([invK[a] @ Y[:, a] for a in range(Y.shape[1])])     # the beta gp_exact_moment forms
    return X, Y, hyper, Z, Sigma, invK, alpha, chol


@pytest.mark.parametrize('case', ['tank', 'syn300'])
def test_em_grad_closed_forms_vs_fourth_order_differences(case):
    X, Y, hyper, Z, Sigma, invK, alpha, chol = _problem(case)
    cl = emo.em_grad_closed(X, hyper, alpha, chol, Z, Sigma)
    fd = emo.em_grad_fd(invK, X, Y, hyper, Z, Sigma)
    assert relinf(cl['dmean_dz'], fd['dmean_dz']) < 1e-5
    assert relinf(cl['dcov_dz'], fd['dcov_dz']) < 1e-5
    assert relinf(emo.sym_pair(cl['dmean_dSigma']), fd['dmean_dSigma']) < 1e-5
    assert relinf(emo.sym_pair(cl['dcov_dSigma']), fd['dcov_dSigma']) < 1e-5
    mean, cov = orc.gp_exact_moment(invK, X, Y, hyper, Z[0], Sigma, extended=True)
    assert relinf(cl['mean'][0], mean) < 1e-10 and relinf(cl['cov'][0], cov) < 1e-4


@pytest.mark.parametrize('scale', ['0.1', '1'])
@pytest.mark.parametrize('Nx', [6, 32])
def test_plain_and_regrouped_em_moments_agree(Nx, scale):
    """The two EM yardsticks of the GPU tests, written independently: the reference's plain formula with its N x N sums in
    long double (gp_exact_moment, extended) and the regrouped closed form (em_grad_closed: backbone through the factor,
    the cross term as written), on one alpha and factor at sn = 0.3, N = 300, Sigma = 0.1 Lambda (correlated) and Lambda.
    They agree to relinf <= 3e-14 on the mean and the covariance."""
    N, Ny = 300, 2
    p = orc.synthetic_problem(N, Nx, Ny, config_id=700 + Nx, H=2)
    X, Y, hyper = p['X'], p['Y'], p['hyper'].copy()
    hyper[:, Nx + 1] = 0.3
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    chol = post['chol']
    invK = np.stack([cho_solve((chol[a], True), np.eye(N)) for a in range(Ny)])
    alpha = np.stack([cho_solve((chol[a], True), Y[:, a]) for a in range(Ny)])
    S = sigmas(hyper, Nx)[scale]
    cl = emo.em_grad_closed(X, hyper, alpha, chol, p['Z'], S)
    for h in range(p['Z'].shape[0]):
        mean, cov = orc.gp_exact_moment(invK, X, Y, hyper, p['Z'][h], S, extended=True, beta=alpha)
        assert relinf(cl['mean'][h], mean) < 3e-14 and relinf(cl['cov'][h], cov) < 3e-14, h


def test_em_grad_limits_as_sigma_vanishes():
    """Sigma -> 0: d mean/dz -> the ME Jacobian, d cov/dz -> diag(d var/dz), d mean/dSigma -> half the mean Hessian,
    d cov[a][b]/dSigma -> the symmetric part of J_a J_b^T (the 'TA' term) plus half the Hessian of var_a on the diagonal."""
    X, Y, hyper, Z, _, invK, alpha, chol = _problem('tank')
    Nx, Ny = X.shape[1], Y.shape[1]
    S = 1e-9 * np.eye(Nx)
    cl = emo.em_grad_closed(X, hyper, alpha, chol, Z, S)
    me = hor.predict_hess(X, hyper, alpha, chol, Z, None, 'ME')
    assert relinf(cl['dmean_dz'], me['dmean']) < 1e-6
    dvar = np.zeros_like(cl['dcov_dz'])
    for a in range(Ny):
        dvar[:, a, a] = me['dvar'][:, a]
    assert relinf(cl['dcov_dz'], dvar) < 1e-5
    assert relinf(cl['dmean_dSigma'], 0.5 * me['hess']) < 1e-5
    J = me['dmean']
    JJ = np.einsum('had,hbe->habde', J, J)
    lim = 0.5 * (JJ + np.swapaxes(JJ, -1, -2))
    for a in range(Ny):
        lim[:, a, a] += 0.5 * me['d2var'][:, a]
    assert relinf(cl['dcov_dSigma'], lim) < 1e-5

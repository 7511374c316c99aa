"""Second derivatives of the prediction without a GPU: the closed-form oracle against central
differences, and the CPU-side metadata of the `jac_jac_gp_b200` CasADi external."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import gp_oracle as orc
from oracle import hess_oracle as hor
from tests._engines import built_lib
from tests._util import load_fixture, relinf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _problem(case):
    if case in ('tank', 'car'):
        m = load_fixture(case); X, Y, hyper = m['X'], m['Y'], m['hyper']
        rng = np.random.default_rng(5)
        Z = X[rng.choice(X.shape[0], 4, replace=False)] + 0.05 * rng.standard_normal((4, X.shape[1]))
        A = rng.standard_normal((X.shape[1],) * 2); Sigma = 1e-3 * np.eye(X.shape[1]) + 1e-4 * A @ A.T
    else:
        p = orc.synthetic_problem(300, 5, 2, config_id=11, H=4)
        X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'], p['Sigma']
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    Sg = np.stack([Sigma * (1 + 0.05 * h) + 1e-5 * h * np.eye(X.shape[1])[::-1] for h in range(Z.shape[0])])   # not symmetric
    return X, hyper, post, Z, Sg


@pytest.mark.parametrize('case', ['tank', 'car', 'syn300'])
def test_predict_hess_closed_forms_vs_central_differences(case):
    X, hyper, post, Z, Sg = _problem(case)
    for method in ('TA', 'ME'):
        hs = hor.predict_hess(X, hyper, post['alpha'], post['chol'], Z, Sg, method)
        fd = hor.predict_hess_fd(X, hyper, post['alpha'], post['chol'], Z, Sg, method)
        assert relinf(hs['d3mean'], fd['d3mean']) < 1e-6
        assert relinf(hs['d2var'], fd['d2var']) < 1e-5
        assert relinf(hs['d2cov'], fd['d2cov']) < 1e-5
        assert np.allclose(hs['d3mean'], np.transpose(hs['d3mean'], (0, 1, 3, 4, 2)), rtol=0, atol=1e-12 * np.abs(hs['d3mean']).max())


def test_predict_grad_closed_vs_fd_oracle():
    """The closed-form first derivatives against predict_grad_fd at the bounds of the existing closed-form check."""
    m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
    Nx = X.shape[1]
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    rng = np.random.default_rng(5)
    Z = X[:3] + 0.05 * rng.standard_normal((3, Nx))
    A = rng.standard_normal((Nx, Nx)); S = 1e-3 * np.eye(Nx) + 1e-4 * A @ A.T
    fd = orc.predict_grad_fd(X, hyper, post['alpha'], post['chol'], Z, S, 'TA')
    cl = hor.predict_grad_closed(X, hyper, post['alpha'], post['chol'], Z, S, 'TA')
    assert relinf(cl['dmean'], fd['dmean']) < 1e-7 and relinf(cl['hess'], fd['hess']) < 1e-6
    assert relinf(cl['dvar'], fd['dvar']) < 1e-5 and relinf(cl['dcov'], fd['dcov']) < 1e-5


JJ_OUT = ['jac_%s_%s' % (o, i) for o in ('jac_mean_z', 'jac_mean_sigma', 'jac_cov_z', 'jac_cov_sigma')
          for i in ('z', 'sigma', 'out_mean', 'out_cov')]


def test_jac_jac_metadata_without_a_gpu():
    L = built_lib(); lib = L.load()
    assert lib.jac_jac_gp_b200_n_in() == 8 and lib.jac_jac_gp_b200_n_out() == 16
    assert [lib.jac_jac_gp_b200_name_in(i) for i in range(8)] == [
        b'z', b'sigma', b'out_mean', b'out_cov', b'out_jac_mean_z', b'out_jac_mean_sigma', b'out_jac_cov_z', b'out_jac_cov_sigma']
    assert [lib.jac_jac_gp_b200_name_out(i).decode() for i in range(16)] == JJ_OUT
    assert lib.jac_jac_gp_b200_name_in(8) is None and lib.jac_jac_gp_b200_name_out(16) is None
    assert not lib.jac_jac_gp_b200_sparsity_in(0) and not lib.jac_jac_gp_b200_sparsity_out(0)     # not bound
    sz = [ctypes.c_longlong(-1) for _ in range(4)]
    assert lib.jac_jac_gp_b200_work(*[ctypes.byref(x) for x in sz]) == 0 and [x.value for x in sz] == [8, 16, 0, 0]


def test_library_exports_every_jac_jac_symbol():
    L = built_lib(); lib = L.load()
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc_casadi.h')).read().split('#ifndef GPMPC_CASADI_H')[1]
    declared = set(re.findall(r'\b(jac_jac_gp_b200[A-Za-z_0-9]*)\s*\(', hdr))
    assert {'jac_jac_gp_b200', 'jac_jac_gp_b200_sparsity_out', 'jac_jac_gp_b200_incref'} <= declared
    assert declared == {s[0] for s in L.SYMBOLS_JAC_JAC}
    for name in declared:
        assert getattr(lib, name) is not None
    assert 'gpmpc_predict_hess' in {s[0] for s in L.SYMBOLS}

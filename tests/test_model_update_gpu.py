"""The model-update entry points on the GPU: a failed rank-1 append keeps its point (Engine.N counts it, and every host
buffer sized by N fits the handle's answers after a refactorisation), and GP.append_data under a prior mean function
equals a GP built on all points."""
import ctypes as C

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._engines import fit
from tests._util import relinf

pytestmark = pytest.mark.gpu


def _singular_problem():
    """Training points 100 length scales apart (K = I up to 2^-1020 terms), sf = 1, sn = 0, so a copy of a training point
    has Schur complement sf2 + sn2 - |L^-1 k|^2 <= 0 in floating point: the K build clamps k(x, x) at sf2 and the ks
    kernel's k(x, x) is exactly sf2 (as in test_append_greedy_gpu)."""
    N = 130
    X = np.column_stack([100.0 * np.arange(N), np.zeros(N)])
    Y = np.random.default_rng(0).standard_normal((N, 2))
    hyper = np.tile([1.0, 1.0, 1.0, 0.0], (2, 1))
    return X, Y, hyper


def test_a_failed_append_keeps_its_point_and_refactorises_on_it():
    X, Y, hyper = _singular_problem()
    N0 = X.shape[0]
    eng = fit(X, Y, hyper, capacity=N0 + 2)
    x_new, y_new = X[5], np.array([0.25, -0.5])
    assert eng.append(x_new, y_new) is False
    # the handle's count, read before anything sizes a host buffer by Engine.N
    n = C.c_int(0)
    assert L.load().gpmpc_get_size(eng.h, C.byref(n), None, None) == L.OK
    assert n.value == N0 + 1 and eng.N == N0 + 1
    assert 'lost positive definiteness' in L.load().gpmpc_last_error(eng.h).decode()
    with pytest.raises(L.GpmpcError) as e:                # the factor is stale until the next factorisation
        eng.get(L.GET_CHOL, 0)
    assert e.value.code == L.ERR_STATE
    info = eng.factorize()                                # the duplicate needs the jitter retry
    assert np.all(info == 1)
    Xa, Ya = np.vstack([X, x_new]), np.vstack([Y, y_new])
    fresh = fit(Xa, Ya, hyper)
    assert np.array_equal(fresh.factorize(), info)
    for a in range(2):
        chol, ref = eng.get(L.GET_CHOL, a), fresh.get(L.GET_CHOL, a)
        assert chol.shape == (N0 + 1, N0 + 1)
        np.testing.assert_allclose(chol, ref, rtol=0, atol=1e-12)
        alpha = eng.get(L.GET_ALPHA, a)
        assert alpha.shape == (N0 + 1,)
        assert relinf(alpha, fresh.get(L.GET_ALPHA, a)) < 1e-6
    mean, var, nlpp = eng.loo()
    fm, fv, fn = fresh.loo()
    assert mean.shape == var.shape == (2, N0 + 1) and nlpp.shape == (2,)
    assert relinf(mean, fm) < 1e-6 and relinf(var, fv) < 1e-6 and relinf(nlpp, fn) < 1e-6


@pytest.mark.parametrize('func', ['const', 'linear'])
def test_append_data_under_a_prior_mean_equals_a_gp_on_all_points(func):
    import gp_mpc_b200
    from gp_mpc_b200 import mean_functions as mf
    N, Nx, Ny = 300, 4, 2
    p = orc.synthetic_problem(N, Nx, Ny, config_id=21)
    hyper = np.hstack([p['hyper'], 0.5 * np.random.default_rng(4).standard_normal((Ny, mf.count_mean_params(func, Nx)))])
    kw = dict(mean_func=func, hyper=dict(hyper=hyper), normalize=False)
    gp = gp_mpc_b200.GP(p['X'][:N - 3], p['Y'][:N - 3], **kw)
    eng = gp.engine
    gp.append_data(p['X'][N - 3:], p['Y'][N - 3:])
    assert gp.engine is eng and eng.N == N                # three rank-1 appends, no refit
    ref = gp_mpc_b200.GP(p['X'], p['Y'], **kw)
    assert relinf(gp.get_chol(), ref.get_chol()) < 1e-10
    assert relinf(gp.get_alpha(), ref.get_alpha()) < 1e-7

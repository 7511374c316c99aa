"""The unscented transform ('UT') on the device: gpmpc_predict(UT) against the numpy recombination of gpmpc_predict(ME) at
the same sigma points and against the CPU oracle, its parameters and argument checks, bit-identity, the device roll-outs
against the host loop of predict(UT) calls, and its accuracy against exact moment matching ('EM')."""
import ctypes

import numpy as np
import pytest
import torch

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import ut_oracle as uto
from tests._engines import fit, problem
from tests._fake_engine import fixture_gp
from tests._util import relinf, trajectories

pytestmark = pytest.mark.gpu

CASES = ['tank', 'car', (300, 1, 1), (300, 1, 9), (400, 8, 1), (400, 8, 9), (500, 17, 1), (500, 17, 9), (300, 32, 1),
         (300, 32, 9)]


def _case_id(c):
    return c if isinstance(c, str) else 'N%d_Nx%d_Ny%d' % c


def _engine(case, **kw):
    X, Y, hyper = problem(case)
    return fit(X, Y, hyper, **kw), X, Y, hyper


def _inputs(hyper, Nx, H, seed):
    """H points near the data and a random full-rank covariance per point, a few tenths of the length scales wide."""
    rng = np.random.default_rng(seed)
    ell = np.abs(hyper[0, :Nx])
    Z = 0.5 * rng.standard_normal((H, Nx))
    G = 0.2 * rng.standard_normal((H, Nx, Nx))
    S = ell[None, :, None] * (G @ np.swapaxes(G, 1, 2) / Nx + 0.01 * np.eye(Nx)) * ell[None, None, :]
    return Z, S


def _sigmas(S, Nx):
    """The covariance layouts of a case: shared and per point full rank, a zero block past the first half (the u-block of
    an open-loop roll-out), and zero."""
    zero_u = S.copy()
    k = max(1, Nx // 2)
    zero_u[:, k:, :] = 0.0; zero_u[:, :, k:] = 0.0
    return {'shared': S[0], 'per_point': S, 'zero_u': zero_u, 'zero': np.zeros((Nx, Nx))}


def _recombined(eng, Z, Sigma, params=uto.DEFAULT_PARAMS):
    """The rule in numpy over gpmpc_predict(ME) at the oracle's sigma points: mean, var, cov, jac and the sums of |terms|
    of mean and cov.  The variance terms are scaled by sf2 (sf2 - |v|^2 cancels in the 'ME' variance)."""
    H, Nx = Z.shape
    P = uto.sigma_points(Z, Sigma, params)
    m, v, _, J = eng.predict(P.reshape(-1, Nx), None, L.METHOD_ME, want_cov=False, want_jac=True)
    m = m.reshape(H, 2 * Nx + 1, -1); v = v.reshape(H, 2 * Nx + 1, -1)
    mean, var, cov = uto.combine(m, v, Nx, params)
    _, wm, wc = uto.weights(Nx, params)
    sf2 = eng.sf2
    d = m - mean[:, None]
    s_mean = np.einsum('k,hka->ha', np.abs(wm), np.abs(m)) + np.abs(m).max(1)
    s_cov = np.einsum('k,hka,hkb->hab', np.abs(wc), np.abs(d), np.abs(d))
    idx = np.arange(m.shape[2])
    s_cov[:, idx, idx] += np.abs(wm).sum() * (np.abs(v).max(1) + sf2[None])
    return mean, var, cov, J.reshape(H, 2 * Nx + 1, m.shape[2], Nx)[:, 0], s_mean, s_cov


def _check(eng, Z, Sigma, params=uto.DEFAULT_PARAMS):
    mean, var, cov, jac = eng.predict(Z, Sigma, L.METHOD_UT)
    rm, rv, rc, rj, s_mean, s_cov = _recombined(eng, Z, Sigma, params)
    idx = np.arange(rm.shape[1])
    assert (np.abs(mean - rm) <= 1e-12 * s_mean).all(), np.max(np.abs(mean - rm) / s_mean)
    assert (np.abs(cov - rc) <= 1e-12 * s_cov).all(), np.max(np.abs(cov - rc) / s_cov)
    assert (np.abs(var - rv) <= 1e-12 * s_cov[:, idx, idx]).all()
    assert np.array_equal(var, np.diagonal(cov, axis1=1, axis2=2))
    assert np.array_equal(cov, np.swapaxes(cov, 1, 2))
    assert np.array_equal(jac, rj)
    return mean, var, cov, jac, s_mean, s_cov


def _with_sf2(eng, hyper):
    eng.sf2 = hyper[:, eng.Nx] ** 2
    return eng


@pytest.mark.parametrize('case', CASES, ids=_case_id)
def test_ut_equals_the_recombination_of_me_at_the_sigma_points(case):
    eng, X, Y, hyper = _engine(case)
    _with_sf2(eng, hyper)
    Nx = X.shape[1]
    H = 50 if Nx == 1 else 7                      # the expanded pass crosses several 64-point chunks
    Z, S = _inputs(hyper, Nx, H, seed=Nx)
    for name, Sigma in _sigmas(S, Nx).items():
        mean, var, cov, jac, s_mean, s_cov = _check(eng, Z, Sigma)
        if name == 'zero':                        # every sigma point is z: 'UT' is 'ME'
            mm, mv, _, mj = eng.predict(Z, None, L.METHOD_ME, want_cov=False)
            idx = np.arange(mm.shape[1])
            assert (np.abs(mean - mm) <= 1e-12 * s_mean).all() and (np.abs(var - mv) <= 1e-12 * s_cov[:, idx, idx]).all()
            # diagonal to the bar: the deviations m_i - mean are rounding-sized here, so the bar of an off-diagonal
            # entry is that of the diagonal entries it sits between
            off = cov.copy(); off[:, idx, idx] = 0.0
            d = np.sqrt(s_cov[:, idx, idx])
            assert (np.abs(off) <= 1e-12 * d[:, :, None] * d[:, None, :]).all()
            assert np.array_equal(jac, mj)
    eng.close()


def test_reserved_handle_after_append_and_remove():
    X, Y, hyper = problem((400, 8, 9))
    eng = _with_sf2(fit(X[:-3], Y[:-3], hyper, capacity=512), hyper)
    eng.append(X[-3], Y[-3]); eng.append(X[-2], Y[-2])
    eng.remove([0, 17])
    Z, S = _inputs(hyper, 8, 9, seed=3)
    _check(eng, Z, S)
    _check(eng, Z, S[2])
    eng.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_parity_with_the_cpu_oracle(name):
    eng, X, Y, hyper = _engine(name)
    Nx = X.shape[1]
    Z, S = _inputs(hyper, Nx, 6, seed=11)
    post = orc.postfit(X, Y, hyper)
    for params in (uto.DEFAULT_PARAMS, (0.5, 2.0, 1.0)):
        eng.set_ut_params(*params)
        for Sigma in (S, S[0]):
            mean, var, cov, jac = eng.predict(Z, Sigma, L.METHOD_UT)
            om, ov, oc, oj = uto.ut_me(X, hyper, post['alpha'], post['chol'], Z, Sigma, params)
            assert relinf(mean, om) < 1e-6 and relinf(var, ov) < 1e-6 and relinf(cov, oc) < 1e-6 and relinf(jac, oj) < 1e-6
    eng.close()


def test_non_default_parameters_and_bad_options():
    eng, X, Y, hyper = _engine((400, 8, 9))
    _with_sf2(eng, hyper)
    Z, S = _inputs(hyper, 8, 5, seed=5)
    for params in ((0.5, 2.0, 1.0), (2.0, 0.0, -3.0), (1.0, 2.0, 0.0)):
        eng.set_ut_params(*params)
        _check(eng, Z, S, params)
    ref = eng.predict(Z, S, L.METHOD_UT)
    lib = eng.lib
    for name, v in (('ut_alpha', 0.0), ('ut_alpha', -1.0), ('ut_kappa', -8.0), ('ut_kappa', -9.5), ('ut_beta', np.nan),
                    ('ut_alpha', np.inf)):
        assert lib.gpmpc_set_option(eng.h, name.encode(), float(v)) == L.ERR_ARG, (name, v)
    for x, y in zip(ref, eng.predict(Z, S, L.METHOD_UT)):     # a rejected option changes nothing
        assert np.array_equal(x, y)
    eng.close()


def test_bits_repeat_and_do_not_depend_on_h_or_the_row():
    eng, X, Y, hyper = _engine((500, 17, 9))
    Z, S = _inputs(hyper, 17, 9, seed=9)
    a = eng.predict(Z, S, L.METHOD_UT)
    b = eng.predict(Z, S, L.METHOD_UT)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    perm = np.array([4, 0, 8, 2, 7, 1, 3, 6, 5])
    c = eng.predict(Z[perm], S[perm], L.METHOD_UT)
    for x, y in zip(a, c):
        assert np.array_equal(x[perm], y)
    for k in (0, 5, 8):
        one = eng.predict(Z[k:k + 1], S[k], L.METHOD_UT)
        for x, y in zip(a, one):
            assert np.array_equal(x[k], y[0])
    eng.close()


def test_device_entry_equals_the_host_entry():
    eng, X, Y, hyper = _engine('tank')
    Z, S = _inputs(hyper, 6, 40, seed=4)
    host = eng.predict(Z, S, L.METHOD_UT)
    dev = torch.device('cuda:0')
    dZ, dS = torch.tensor(Z, device=dev), torch.tensor(S, device=dev)
    out = [torch.empty(sh, dtype=torch.float64, device=dev) for sh in ((40, 4), (40, 4), (40, 4, 4), (40, 4, 6))]
    eng.predict_device(L.METHOD_UT, 40, dZ.data_ptr(), dS.data_ptr(), 1, *[o.data_ptr() for o in out], sync=True)
    for x, y in zip(host, out):
        assert np.array_equal(x, y.cpu().numpy())
    with pytest.raises(L.GpmpcError) as e:
        eng.predict_device(L.METHOD_UT, 40, dZ.data_ptr(), None, 1, *[o.data_ptr() for o in out], sync=True)
    assert e.value.code == L.ERR_ARG
    eng.close()


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_rollouts_equal_the_host_loop(name):
    """GP.rollout(methods=['UT']) on the device (gpmpc_rollout for one open-loop trajectory, gpmpc_rollout_batch for a batch,
    open loop and with feedback) equals the host loop of predict(UT) calls; gpmpc_rollout is the batch of one bit for bit."""
    gp, m = fixture_gp(name)
    X0, U, x_ref = trajectories(name, 5, 6, cyclic=False)
    for kw in (dict(), dict(feedback=True, x_ref=x_ref)):
        rm, rv = gp.rollout(X0, U, methods=['UT', 'TA'], **kw)
        hm, hv = gp.rollout(X0, U, methods=['UT', 'TA'], device_rollout=False, **kw)
        for b in range(5):
            assert relinf(rm[:, b], hm[:, b]) < 1e-12 and relinf(rv[:, b], hv[:, b]) < 1e-12, (kw, b)
        # 'UT' runs first from a positive semidefinite covariance (with feedback 'TA' then inherits its u-blocks)
        assert (rv[0, :, 1:] > 0).all()
    sm, sv = gp.rollout(X0[0], U[0], methods=['UT'])
    hm, hv = gp.rollout(X0[0], U[0], methods=['UT'], device_rollout=False)
    assert relinf(sm, hm) < 1e-12 and relinf(sv, hv) < 1e-12
    eng = gp.engine
    Ny, Nx = X0.shape[1], eng.Nx
    z0 = np.concatenate([X0, U[:, 0]], 1) if not m['normalize'] else np.concatenate(
        [(X0 - m['meta']['meanX']) / m['meta']['stdX'], (U[:, 0] - m['meta']['meanU']) / m['meta']['stdU']], 1)
    S = np.tile(np.eye(Nx) * 1e-6, (5, 1, 1))
    S[:, :Ny, :Ny] = np.diag(m['hyper'][:, -1] ** 2)
    a = eng.rollout(z0[0], U[0], S[0], L.METHOD_UT)
    b = eng.rollout_batch(z0[:1], U[:1], S[:1], L.METHOD_UT)
    for x, y in zip(a, b):
        assert np.array_equal(x, y[0])
    c1 = eng.rollout_batch(z0, U, S, L.METHOD_UT)
    c2 = eng.rollout_batch(z0, U, S, L.METHOD_UT)
    for k, (x, y) in enumerate(zip(c1, c2)):
        assert np.array_equal(x, y)
        assert np.array_equal(x[3], eng.rollout_batch(z0[3:4], U[3:4], S[3:4], L.METHOD_UT)[k][0])
    gp.close()


def test_accuracy_against_exact_moment_matching():
    """One step on the tank fixture: quartering Sigma cuts |UT - EM| of the mean by at least 8x (O(sigma^4)) and |TA - EM|
    by about 4x (O(sigma^2))."""
    eng, X, Y, hyper = _engine('tank')
    z = np.array([[0.3, -0.2, 0.1, 0.4, -0.5, 0.2]])
    base = np.diag(hyper[0, :6] ** 2) * 0.003
    ut_err, ta_err = [], []
    for s2 in (1.0, 0.25, 0.0625):
        Sigma = base * s2
        em = eng.predict(z, Sigma, L.METHOD_EM, want_jac=False)[0]
        ut = eng.predict(z, Sigma, L.METHOD_UT)[0]
        ta = eng.predict(z, Sigma, L.METHOD_TA)[0]
        ut_err.append(np.abs(ut - em).max()); ta_err.append(np.abs(ta - em).max())
    for k in range(2):
        assert ut_err[k] / ut_err[k + 1] >= 8, ut_err
        assert 3.5 < ta_err[k] / ta_err[k + 1] < 4.5, ta_err
    assert ut_err[0] < 0.1 * ta_err[0]
    eng.close()


def test_argument_and_state_checks():
    eng, X, Y, hyper = _engine('tank')
    lib = eng.lib
    H, Nx, Ny = 3, 6, 4
    Z, S = _inputs(hyper, Nx, H, seed=1)
    dp = ctypes.POINTER(ctypes.c_double)
    buf = lambda *sh: np.zeros(sh)
    p = lambda a: a.ctypes.data_as(dp)
    with pytest.raises(L.GpmpcError) as e:                  # Sigma is required
        eng.predict(Z, None, L.METHOD_UT)
    assert e.value.code == L.ERR_ARG
    assert lib.gpmpc_predict_grad(eng.h, L.METHOD_UT, H, p(Z), p(S), 1, p(buf(H, Ny)), p(buf(H, Ny)), p(buf(H, Ny, Ny)),
                                  p(buf(H, Ny, Nx)), p(buf(H, Ny, Nx)), p(buf(H, Ny, Ny, Nx)), None) == L.ERR_ARG
    assert lib.gpmpc_predict_hess(eng.h, L.METHOD_UT, H, p(Z), p(S), 1, *[None] * 10) == L.ERR_ARG
    Nt = 3
    z0, S0 = Z[:1], S[:1]
    U = np.zeros((1, Nt, 2))
    outs = [buf(1, Nt, Ny), buf(1, Nt, Ny), buf(1, Ny, Ny), buf(1, Nt, Ny, Nx + 2 * (Nt - 1)), buf(1, Nt, Ny, Nx + 2 * (Nt - 1))]
    assert lib.gpmpc_rollout_batch_grad(eng.h, L.METHOD_UT, 1, Nt, p(z0), p(U), p(S0), None, None, None, None,
                                        *[p(o) for o in outs]) == L.ERR_ARG
    assert lib.gp_b200_bind(eng.h, L.METHOD_UT, 2) == L.ERR_ARG
    lib.gp_b200_unbind()
    assert lib.gpmpc_rollout_batch(eng.h, L.METHOD_UT, 1, Nt, p(z0), p(U), None, None, None, None, None,
                                   *[p(o) for o in outs[:3]]) == L.ERR_ARG           # a NULL Sigma0
    assert lib.gpmpc_predict(eng.h, 4, H, p(Z), p(S), 1, *[None] * 4) == L.ERR_ARG  # still an unknown method
    eng.close()
    part = L.Engine(X.shape[0], Nx, Ny, out_begin=1, out_count=2, device=0)     # owns outputs 1 and 2 only
    part.set_data(X, Y); part.set_hyper(hyper); part.factorize()
    with pytest.raises(L.GpmpcError) as e:
        part.predict(Z, S, L.METHOD_UT)
    assert e.value.code == L.ERR_STATE
    assert lib.gpmpc_rollout(part.h, L.METHOD_UT, Nt, p(z0[0]), p(U[0]), p(S0[0]), None,
                             *[p(o) for o in outs[:3]]) == L.ERR_STATE
    part.close()

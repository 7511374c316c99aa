"""gpmpc_rollout_sample_grad on the device (DESIGN 4.16): the draws against gpmpc_rollout_sample bit for bit, step 1
against gpmpc_predict_grad, the derivatives against central differences of gpmpc_rollout_sample and against the forward-mode
checker tests/_sample_grad_oracle.py, a model whose draws drop points, bit-identity across rows, batches and repeats,
error codes, and the gradient of a Monte Carlo objective through GP.sample_rollout_grad."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import sample_oracle as so
from tests import _sample_grad_oracle as sgo
from tests._engines import sample_engine
from tests._util import load_fixture, load_golden

pytestmark = pytest.mark.gpu

# Central-difference step and bar relative to 1 + max |derivative| (DESIGN 4.16): the quotient's error is the draw's
# rounding over the step; R^-1 enters twice and tank's pivots are small, so tank needs a wider step than the synthetic case
STEP = dict(synthetic=1e-6, tank=1e-4)
BAR = dict(synthetic=2e-5, tank=5e-6)
# the device against the checker, relative to 1 + max |derivative|: two different roundings of the same recursion,
# amplified by R^-1 twice on tank's small pivots
ORACLE_BAR = dict(synthetic=1e-7, tank=1e-5)


def _inputs(m, B, Nt, seed, spread=0.3):
    """Starts spread around the data and open-loop inputs, GP input units, and the draws' normals eps and xi."""
    rng = np.random.default_rng(seed)
    X = m['X']
    Nx, Ny = X.shape[1], m['Y'].shape[1]
    z0 = X[rng.integers(0, X.shape[0], B)] + spread * X.std(0) * rng.standard_normal((B, Nx))
    U = np.repeat(z0[:, None, Ny:], Nt, 1) + spread * X.std(0)[Ny:] * rng.standard_normal((B, Nt, Nx - Ny))
    return z0, U, rng.standard_normal((B, Nt, Ny)), rng.standard_normal((B, Nt, Ny))


def _factor(eng, m):
    Ny = m['Y'].shape[1]
    Linv = np.stack([eng.get(L.GET_LINV, a) for a in range(Ny)])
    model = dict(X=m['X'], hyper=m['hyper'], alpha=np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)]),
                 chol=np.stack([np.linalg.inv(Li) for Li in Linv]))
    return model, Linv


def _perturbed(z0, U, K, p, h):
    z0, U = z0.copy(), U.copy()
    K = None if K is None else K.copy()
    Nx = z0.shape[1]
    if p < Nx:
        z0[:, p] += h
    elif K is None:
        Nu = U.shape[2]
        U[:, 1 + (p - Nx) // Nu, (p - Nx) % Nu] += h
    else:
        K.reshape(-1)[p - Nx] += h
    return z0, U, K


@pytest.mark.parametrize('B', [1, 64, 65, 130])
def test_draws_are_rollout_sample_bit_for_bit(B):
    eng, m = sample_engine('synthetic')
    z0, U, eps, xi = _inputs(m, B, 6, B)
    Ny, Nx = m['Y'].shape[1], m['X'].shape[1]
    K = 0.1 * np.random.default_rng(B).standard_normal((Nx - Ny, Ny))
    for args in ((z0, U, eps), (z0, U, eps, xi), (z0, U, eps, xi, None, K, np.full(Ny, 0.1))):
        ref = eng.rollout_sample(*args)
        got = eng.rollout_sample_grad(*args)
        for x, y in zip(ref, got[:3]):
            assert np.array_equal(x, y)
        assert np.isfinite(got[3]).all()
    eng.close()


@pytest.mark.parametrize('name', ['synthetic', 'tank'])
def test_step_one_against_predict_grad(name):
    """df_0 = J dz + (dvar_dz . dz) / (2 sqrt(var)) eps_0 on the unit columns of z0."""
    eng, m = sample_engine(name)
    B = 70
    z0, U, eps, _ = _inputs(m, B, 1, 2)
    _, _, kept, D = eng.rollout_sample_grad(z0, U, eps)
    assert kept.all()
    g = eng.predict_grad(z0, None, L.METHOD_ME)
    want = g['jac'] + g['dvar_dz'] / (2 * np.sqrt(g['var']))[..., None] * eps[:, 0, :, None]
    assert np.abs(D[:, 0] - want).max() <= 1e-10 * (1 + np.abs(want).max())
    eng.close()


# tank's paths spread over the whole data set: near the data its conditional variances come within the margin of the delta
# rule after a few steps, and under feedback they converge onto the reference (both are covered on the host)
SPREAD = dict(synthetic=0.3, tank=1.0)


@pytest.mark.parametrize('name, feedback', [('synthetic', False), ('synthetic', True), ('tank', False)])
def test_central_differences_on_the_device(name, feedback):
    eng, m = sample_engine(name)
    Nt = 12 if name == 'synthetic' else 5
    Ny, Nx = m['Y'].shape[1], m['X'].shape[1]
    z0, U, eps, xi = _inputs(m, 2, Nt, 5, SPREAD[name])
    K = 0.05 * np.random.default_rng(1).standard_normal((Nx - Ny, Ny)) if feedback else None
    x_ref = np.full(Ny, 0.1) if feedback else None
    s, z_out, kept, D = eng.rollout_sample_grad(z0, U, eps, xi, None, K, x_ref)
    model, Linv = _factor(eng, m)
    sgo.assert_margin(sgo.rollout_sample_grad(model, Linv, z0, U, eps, xi, None, K, x_ref)['d'], m['hyper'])
    h = STEP[name]
    for p in range(D.shape[-1]):
        sp = eng.rollout_sample(*_perturbed(z0, U, K, p, h)[:2], eps, xi, None, _perturbed(z0, U, K, p, h)[2], x_ref)
        sm = eng.rollout_sample(*_perturbed(z0, U, K, p, -h)[:2], eps, xi, None, _perturbed(z0, U, K, p, -h)[2], x_ref)
        assert np.array_equal(sp[2], kept) and np.array_equal(sm[2], kept)
        fd = (sp[0] - sm[0]) / (2 * h)
        assert np.abs(D[..., p] - fd).max() / (1 + np.abs(D).max()) < BAR[name], p
    eng.close()


@pytest.mark.parametrize('lapack', [False, True])
@pytest.mark.parametrize('name', ['synthetic', 'tank'])
def test_against_the_checker(name, lapack):
    """The device against the numpy recursion on the engine's own L^-1 and alpha, or on a LAPACK factor."""
    eng, m = sample_engine(name)
    z0, U, eps, xi = _inputs(m, 3, 8 if name == 'synthetic' else 5, 7, SPREAD[name])
    s, z_out, kept, D = eng.rollout_sample_grad(z0, U, eps, xi)
    if lapack:
        post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
        model = dict(X=m['X'], hyper=m['hyper'], alpha=post['alpha'], chol=post['chol'])
        Linv = np.stack([np.linalg.inv(c) for c in post['chol']])
    else:
        model, Linv = _factor(eng, m)
    r = sgo.rollout_sample_grad(model, Linv, z0, U, eps, xi)
    assert np.array_equal(r['kept'], kept)
    err = np.abs(D - r['dsamples']).max() / (1 + np.abs(r['dsamples']).max())
    assert err < ORACLE_BAR[name] * (10 if lapack else 1), err
    eng.close()


def test_a_model_whose_draws_drop_points():
    """x+ = 0.5 x: every draw converges to a fixed point of its function, later points leave the conditioning set, and
    the derivatives stay finite and follow the branch the draw took."""
    import gp_mpc_b200
    rng = np.random.default_rng(2)
    X = rng.uniform(-2, 2, (60, 2))
    Y = 0.5 * X + 1e-3 * rng.standard_normal(X.shape)
    hyper = np.array([[3.0, 3.0, 1.0, 1e-3], [3.0, 3.0, 1.0, 1e-3]])
    eng = gp_mpc_b200.Engine(60, 2, 2, device=0)
    eng.set_data(X, Y); eng.set_hyper(hyper); eng.factorize()
    B, Nt = 4, 40
    z0 = rng.uniform(-1.5, 1.5, (B, 2))
    eps = rng.standard_normal((B, Nt, 2))
    s, z_out, kept, D = eng.rollout_sample_grad(z0, np.zeros((B, Nt, 0)), eps)
    assert (kept == 0).any() and np.isfinite(D).all()
    model, Linv = _factor(eng, dict(X=X, Y=Y, hyper=hyper))
    r = sgo.rollout_sample_grad(model, Linv, z0, np.zeros((B, Nt, 0)), eps)
    assert np.array_equal(r['kept'], kept)
    assert np.abs(D - r['dsamples']).max() <= 1e-6 * (1 + np.abs(r['dsamples']).max())
    eng.close()


def test_bit_identical_alone_in_a_batch_and_on_repeat():
    eng, m = sample_engine('synthetic')
    z0, U, eps, xi = _inputs(m, 130, 6, 3)
    full = eng.rollout_sample_grad(z0, U, eps, xi)
    again = eng.rollout_sample_grad(z0, U, eps, xi)
    for x, y in zip(full, again):
        assert np.array_equal(x, y)
    for b in (0, 63, 64, 129):
        one = eng.rollout_sample_grad(z0[b:b + 1], U[b:b + 1], eps[b:b + 1], xi[b:b + 1])
        for x, y in zip(full, one):
            assert np.array_equal(x[b:b + 1], y)
    eng.close()


def test_error_codes_leave_the_model_usable():
    import gp_mpc_b200
    eng, m = sample_engine('synthetic')
    z0, U, eps, _ = _inputs(m, 2, 4, 1)
    Ny, Nx = m['Y'].shape[1], m['X'].shape[1]
    h = eng.h
    dp = lambda a: a.ctypes.data_as(L._dp) if a is not None else None
    out = [np.empty((2, 4, Ny)), np.empty((2, 4, Nx)), np.empty((2, 4, Ny), dtype=np.int32), np.empty((2, 4, Ny, Nx + 3 * 2))]
    lib = L.load()
    ip = out[2].ctypes.data_as(L._ip)
    assert lib.gpmpc_rollout_sample_grad(h, 2, 4, dp(z0), dp(U), dp(eps), None, None, None, None, None, dp(out[0]),
                                         dp(out[1]), ip, None) == L.ERR_ARG
    assert lib.gpmpc_rollout_sample_grad(h, 0, 4, dp(z0), dp(U), dp(eps), None, None, None, None, None, dp(out[0]),
                                         dp(out[1]), ip, dp(out[3])) == L.ERR_ARG
    Nt = 65
    z0b, Ub, epsb, _ = _inputs(m, 1, Nt, 1)
    big = np.empty((1, Nt, Ny, Nx + (Nt - 1) * 2))
    assert lib.gpmpc_rollout_sample_grad(h, 1, Nt, dp(z0b), dp(Ub), dp(epsb), None, None, None, None, None,
                                         dp(np.empty((1, Nt, Ny))), None, None, dp(big)) == L.ERR_ARG
    assert b'Nt' in lib.gpmpc_last_error(h)
    ref = eng.rollout_sample(z0, U, eps)
    got = eng.rollout_sample_grad(z0, U, eps)
    assert all(np.array_equal(x, y) for x, y in zip(ref, got[:3]))
    fresh = gp_mpc_b200.Engine(m['X'].shape[0], Nx, Ny, device=0)
    fresh.set_data(m['X'], m['Y']); fresh.set_hyper(m['hyper'])
    assert lib.gpmpc_rollout_sample_grad(fresh.h, 2, 4, dp(z0), dp(U), dp(eps), None, None, None, None, None,
                                               dp(out[0]), dp(out[1]), ip, dp(out[3])) == L.ERR_STATE
    fresh.close()
    eng.close()


def test_gradient_of_a_monte_carlo_objective():
    """J(x0) = mean over 256 draws of sum_t |x_t - x_ref|^2 through GP.sample_rollout_grad, against its difference
    quotient with the same seed."""
    import gp_mpc_b200
    m = load_fixture('tank')
    d = load_golden('derived', 'tank')
    gp = gp_mpc_b200.GP(m['X'], m['Y'], mean_func='zero', gp_method='TA', normalize=True, hyper=dict(hyper=m['hyper']),
                        meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    x0, u0 = np.asarray(d['x0'], dtype=np.float64), np.asarray(d['u0'], dtype=np.float64)
    U = np.tile(u0, (5, 1))
    x_ref = 0.9 * x0
    Sigma0 = np.diag(np.r_[np.full(4, 1e-2), np.full(2, 1e-6)])

    def objective(x):
        s = gp.sample_rollout(x, U, 256, seed=3, Sigma0=Sigma0)
        return np.mean(np.sum((s[:, 1:] - x_ref) ** 2, axis=(1, 2)))
    r = gp.sample_rollout_grad(x0, U, 256, seed=3, Sigma0=Sigma0)
    s = r['samples']
    grad = np.mean(np.einsum('ntk,ntkj->nj', 2 * (s[:, 1:] - x_ref), r['dsamples_dx0'][:, 1:]), axis=0)
    fd = np.empty(4)
    for j in range(4):
        h = 1e-4 * (abs(x0[j]) + 1)
        xp, xm = x0.copy(), x0.copy()
        xp[j] += h
        xm[j] -= h
        fd[j] = (objective(xp) - objective(xm)) / (2 * h)
    assert np.abs(grad - fd).max() <= 1e-4 * (1 + np.abs(fd).max()), (grad, fd)
    gp.close()

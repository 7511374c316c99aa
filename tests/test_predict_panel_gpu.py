"""The predict product reads L^-1 from its panel copy (dLiP, predict_streamk.cuh), refreshed from the first row each writer
of L^-1 touched.  A band the refresh missed still holds the old factor's rows, which changes var by O(1); so after every
writer var is compared with sf2 - |L^-1 ks|^2 formed in long double from GET_LINV and the kernel on the engine's data,
normalised by sf2 + (|L^-1| |ks|)^2 (the sum of |terms|, including the cancellation inside L^-1 ks).  Two paths see the
product: gpmpc_predict (all outputs) and gpmpc_posterior_cov (diagonal, also on a sharded handle).

Writers: factorize, set_hyper + factorize, set_data + factorize (GP.replace_data_all), the jitter re-run of one output,
append into the reserve and across a 256-row tile border, append_greedy, remove at 0, mid and N - 1, a sliding window,
and a sharded handle (out_begin = 1).  Shapes: Npad / 128 odd (the half tile) and even, N < 256, Ny in {1, 3, 8},
H in {1, 50, 65} (65: two chunks).  The other products of L^-1 (predict_grad, predict_hess, roll-outs, the refinement)
must repeat their bits and, for the derivatives, agree with the long-double reference within the bars of
test_predict_derivs_shapes_gpu."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import hess_oracle as hor
from tests._util import PREDICT_TOL, PREDICT_VAR_TOL, normalised

pytestmark = pytest.mark.gpu

LD = np.longdouble
HS = (1, 50, 65)


def problem(N, Nx, Ny, seed=0, sn=0.1):
    p = orc.synthetic_problem(N, Nx, Ny, config_id=700 + 11 * Nx + Ny + seed)
    hyper = p['hyper'].copy()
    hyper[:, Nx + 1] = sn
    return p['X'], p['Y'], hyper


def engine(X, Y, hyper, cap=None, out_begin=0, out_count=None):
    eng = L.Engine(X.shape[0], X.shape[1], Y.shape[1], device=0, capacity=cap, out_begin=out_begin,
                      out_count=out_count)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)
    eng.factorize()
    return eng


def points(X, H, seed):
    rng = np.random.default_rng(seed)
    return X[rng.integers(0, X.shape[0], H)] + 0.1 * rng.standard_normal((H, X.shape[1]))


def var_ref(eng, X, hyper, Z):
    """(ref, scale), each (H, out_count): sf2 - |L^-1 ks|^2 and sf2 + (|L^-1| |ks|)^2 in long double."""
    Nx = X.shape[1]
    ref, scale = [], []
    for a in eng.local_outputs:
        ell, sf2 = LD(1) * hyper[a, :Nx], LD(hyper[a, Nx]) ** 2
        d = (X.astype(LD)[:, None, :] - Z.astype(LD)[None, :, :]) / ell
        ks = sf2 * np.exp(-0.5 * np.sum(d * d, axis=2))                       # (N, H)
        Li = eng.get(L.GET_LINV, a).astype(LD)
        v = Li @ ks
        ref.append(sf2 - np.sum(v * v, axis=0))
        scale.append(sf2 + np.sum((np.abs(Li) @ ks) ** 2, axis=0))
    return np.stack(ref, 1), np.stack(scale, 1)


def check(eng, X, hyper, label, hs=HS):
    """var of gpmpc_predict (all outputs on the handle) and the diagonal of gpmpc_posterior_cov against var_ref."""
    full = eng.out_begin == 0 and eng.out_count == eng.Ny
    Zs = [points(X, H, seed=H + X.shape[0]) for H in hs]
    ref_all, scale_all = var_ref(eng, X, hyper, np.vstack(Zs))
    for H, Z, o in zip(hs, Zs, np.cumsum([0] + list(hs))):
        ref, scale = ref_all[o:o + H], scale_all[o:o + H]
        got = {}
        if full:
            _, v1, _, _ = eng.predict(Z, 1e-4 * np.eye(X.shape[1]), L.METHOD_TA)
            _, v2, _, _ = eng.predict(Z, 1e-4 * np.eye(X.shape[1]), L.METHOD_TA)
            assert np.array_equal(v1, v2), (label, H)
            got['predict'] = v1
        got['posterior_cov'] = np.stack([np.diag(c) for c in eng.posterior_cov(Z)], 1)
        for k, v in got.items():
            err = float(np.max(np.abs(v.astype(LD) - ref) / scale))
            print('MEASURED', label, k, 'H=%d' % H, '%.2e' % err)
            assert err <= PREDICT_VAR_TOL, (label, k, H, err)


# name -> (N, Nx, Ny): Npad / 128 = 2 (N < 256), 3 (half tile), 5, 6
SHAPES = {'n200_ny1': (200, 4, 1), 'n300_ny3': (300, 5, 3), 'n600_ny8': (600, 6, 8), 'n700_ny3': (700, 3, 3)}


@pytest.mark.parametrize('name', list(SHAPES))
def test_factorize_and_refit(name):
    N, Nx, Ny = SHAPES[name]
    X, Y, hyper = problem(N, Nx, Ny)
    eng = engine(X, Y, hyper)
    check(eng, X, hyper, name + ' factorize')
    hyper2 = hyper.copy()
    hyper2[:, :Nx] *= 0.8
    eng.set_hyper(hyper2)
    eng.factorize()
    check(eng, X, hyper2, name + ' set_hyper')
    X2, Y2, _ = problem(N, Nx, Ny, seed=1)                 # GP.replace_data_all: set_data + factorize
    eng.set_data(X2, Y2)
    eng.factorize()
    check(eng, X2, hyper2, name + ' replace_data')


def test_jitter_rerun_of_one_output():
    """Output 1 of 3 has duplicated points and sn = 1e-10: gpmpc_factorize re-runs it with the jitter."""
    N, Nx = 300, 4
    X, Y, hyper = problem(N, Nx, 3)
    eng = engine(X, Y, hyper)
    check(eng, X, hyper, 'before jitter', hs=(50,))
    X2 = X.copy()
    X2[N // 2:] = X2[:N - N // 2]
    hyper[1, Nx + 1] = 1e-10
    eng.set_data(X2, Y)
    eng.set_hyper(hyper)
    assert list(eng.factorize()) == [0, 1, 0]
    check(eng, X2, hyper, 'jitter re-run')


@pytest.mark.parametrize('Ny', [1, 3, 8])
def test_append_into_the_reserve_and_across_a_tile_border(Ny):
    Nx = 4
    X, Y, hyper = problem(262, Nx, Ny)
    eng = engine(X[:250], Y[:250], hyper, cap=600)
    check(eng, X[:250], hyper, 'fit 250', hs=(50,))
    for n in range(250, 253):
        assert eng.append(X[n], Y[n])
    check(eng, X[:253], hyper, 'append to 253', hs=(1, 50))
    for n in range(253, 262):                               # rows 253 .. 261 cross the 256-row tile border
        assert eng.append(X[n], Y[n])
    check(eng, X[:262], hyper, 'append to 262')


def test_append_greedy():
    Nx, Ny = 4, 3
    X, Y, hyper = problem(500, Nx, Ny)
    eng = engine(X[:240], Y[:240], hyper, cap=512)
    check(eng, X[:240], hyper, 'fit 240', hs=(50,))
    picked, _, ok = eng.append_greedy(X[240:], Y[240:], 30)
    assert ok and len(picked) == 30
    Xn = np.vstack([X[:240], X[240:][picked]])
    check(eng, Xn, hyper, 'append_greedy')


def test_remove_at_the_ends_and_mid_and_a_sliding_window():
    Nx, Ny = 4, 3
    X, Y, hyper = problem(420, Nx, Ny)
    N = 400
    eng = engine(X[:N], Y[:N], hyper, cap=512)
    Xc, Yc = X[:N], Y[:N]
    check(eng, Xc, hyper, 'fit 400', hs=(50,))
    for where, pick in (('0', lambda n: 0), ('mid', lambda n: n // 2), ('N-1', lambda n: n - 1)):
        i = pick(Xc.shape[0])
        eng.remove([i])
        Xc, Yc = np.delete(Xc, i, 0), np.delete(Yc, i, 0)
        check(eng, Xc, hyper, 'remove ' + where, hs=(1, 50))
    for n in range(N, N + 4):                               # window: drop the oldest, append the newest
        eng.remove([0])
        assert eng.append(X[n], Y[n])
        Xc, Yc = np.vstack([Xc[1:], X[n]]), np.vstack([Yc[1:], Y[n]])
        check(eng, Xc, hyper, 'window %d' % n, hs=(50,))


def test_sharded_handle():
    """Outputs 1 and 2 of 3 on one handle (out_begin = 1): the panel is per owned output."""
    Nx, Ny = 4, 3
    X, Y, hyper = problem(330, Nx, Ny)
    eng = engine(X[:300], Y[:300], hyper, cap=400, out_begin=1, out_count=2)
    check(eng, X[:300], hyper, 'sharded fit')
    for n in range(300, 330):
        assert eng.append(X[n], Y[n])
    check(eng, X[:330], hyper, 'sharded append', hs=(50,))
    eng.remove([5])
    check(eng, np.delete(X[:330], 5, 0), hyper, 'sharded remove', hs=(50,))


def test_other_products_of_linv():
    """predict_grad / predict_hess repeat their bits and match the long-double reference; roll-outs repeat their bits;
    the refinement (two L^-1 products and one of L) matches var_ref."""
    Nx, Ny = 5, 3
    X, Y, hyper = problem(300, Nx, Ny)
    eng = engine(X[:290], Y[:290], hyper, cap=400)
    for n in range(290, 300):                               # the panel after an append, not just a factorisation
        assert eng.append(X[n], Y[n])
    alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)])
    linv = np.stack([eng.get(L.GET_LINV, a) for a in range(Ny)])
    Z = points(X, 6, seed=3)
    S = 1e-3 * np.eye(Nx)
    ref = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, 'TA')
    ab = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, 'TA', absolute=True)
    g1, g2 = eng.predict_grad(Z, S, L.METHOD_TA), eng.predict_grad(Z, S, L.METHOD_TA)
    h1, h2 = eng.predict_hess(Z, S, L.METHOD_TA), eng.predict_hess(Z, S, L.METHOD_TA)
    for out, other, keys in ((g1, g2, ('var', 'dvar_dz', 'dcov_dz')), (h1, h2, ('var', 'dvar_dz', 'd2var_dz2'))):
        for k in out:
            assert np.array_equal(out[k], other[k]), k
        for k in keys:
            err = normalised(out[k], ref[k], ab[k])
            print('MEASURED', k, '%.2e' % err)
            assert err <= PREDICT_TOL[k], (k, err)
    Nu = Nx - Ny
    z0 = np.tile(X[:1], (4, 1))
    U = 0.1 * np.ones((4, 5, Nu))
    S0 = np.tile(1e-4 * np.eye(Nx), (4, 1, 1))
    r1, r2 = eng.rollout_batch(z0, U, S0, L.METHOD_TA), eng.rollout_batch(z0, U, S0, L.METHOD_TA)
    for a, b in zip(r1, r2):
        assert np.array_equal(a, b)
    eng.set_option('refine', 1)
    check(eng, X, hyper, 'refine', hs=(1, 65))

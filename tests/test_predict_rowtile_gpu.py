"""The predict product in 256-row tiles: sizes whose Npad / 128 is odd end in a 128-row half tile (N = 1100: Npad 1152;
N = 100: one half tile and nothing else).  var matches sf2 - |L^-1 ks|^2, a point's var / cov do not depend on its row
or the batch size, the refinement path and predict_grad (whose second product runs over the upper triangle, with a
shorter k-step list than the lower one at these sizes) agree with the oracle, and repeat calls are bit-identical at
any persistent-grid size."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._engines import synthetic_engine
from tests._util import relinf


pytestmark = pytest.mark.gpu

POOL = 130
SIZES = [(1100, 1), (1100, 8), (100, 1), (100, 8)]


@pytest.mark.parametrize('N,Ny', SIZES)
def test_half_tile_var_matches_linv_ks(N, Ny):
    eng, p = synthetic_engine(N, 6, Ny, seed=31 + N + Ny, H=POOL)
    X, Z, hyper = p['X'], p['Z'], p['hyper']
    for H in (1, 56, 130):
        _, var, _, _ = eng.predict(Z[:H], None, L.METHOD_ME, want_cov=False, want_jac=False)
        for a in range(Ny):
            sf2 = hyper[a, 6] ** 2
            v = eng.get(L.GET_LINV, a) @ orc.covSEard(X, Z[:H], hyper[a, :6], sf2)
            assert np.abs(var[:, a] - (sf2 - np.einsum('nh,nh->h', v, v))).max() < 1e-10 * sf2, (H, a)
    eng.close()


@pytest.mark.parametrize('N,Ny', SIZES)
def test_half_tile_results_do_not_depend_on_batch_or_row(N, Ny):
    eng, p = synthetic_engine(N, 6, Ny, seed=57 + N + Ny, H=POOL)
    Z, Sigma = p['Z'], p['Sigma']
    _, var_ref, cov_ref, _ = eng.predict(Z, Sigma, L.METHOD_TA)
    rng = np.random.default_rng(N + Ny)
    for H in (1, 8, 9, 50, 64, 65, 130):
        idx = rng.permutation(POOL)[:H]
        _, var, cov, _ = eng.predict(Z[idx], Sigma, L.METHOD_TA)
        assert np.array_equal(var, var_ref[idx]), H
        assert np.array_equal(cov, cov_ref[idx]), H
    eng.close()


@pytest.mark.parametrize('N,Ny', SIZES)
def test_half_tile_refine_and_grad_vs_oracle(N, Ny):
    eng, p = synthetic_engine(N, 6, Ny, seed=83 + N + Ny, H=POOL)
    X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'][:9], p['Sigma']
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], Z)
    Jo = orc.gp_mean_jac(X, hyper, post['alpha'], Z)
    mean, var, cov, jac = eng.predict(Z, Sigma, L.METHOD_TA)
    assert relinf(mean, mo) < 1e-6 and relinf(var, vo) < 1e-6 and relinf(jac, Jo) < 1e-6
    assert relinf(cov, orc.ta_cov(vo, Jo, Sigma)) < 1e-6
    eng.set_option('refine', 1)
    mean_r, var_r, _, _ = eng.predict(Z, Sigma, L.METHOD_TA)
    assert relinf(var_r, vo) < 1e-6 and relinf(mean_r, mo) < 1e-6
    eng.set_option('refine', 0)
    g = eng.predict_grad(Z, Sigma, L.METHOD_TA)
    assert np.array_equal(g['var'], var) and np.array_equal(g['cov'], cov)
    fd = orc.predict_grad_fd(X, hyper, post['alpha'], post['chol'], Z, Sigma, 'TA')
    assert relinf(g['jac'], fd['dmean']) < 1e-5
    assert relinf(g['dvar_dz'], fd['dvar']) < 1e-5
    assert relinf(g['dcov_dz'], fd['dcov']) < 1e-5
    eng.close()


@pytest.mark.parametrize('N', [1000, 1100])
def test_refine_after_a_full_k_build_vs_oracle(N):
    """A full K build (PROF_KBUILD_FULL) leaves K's upper triangle in output 0's L slab and the factorisation rewrites only
    the lower one: the refinement's product with L must not read the 128 x 128 blocks above the diagonal."""
    import gp_mpc_b200
    p = orc.synthetic_problem(N, 6, 2, config_id=11, H=POOL)
    X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'], p['Z'][:20], p['Sigma']
    eng = gp_mpc_b200.Engine(N, 6, 2, device=0)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)
    eng.profile(L.PROF_KBUILD_FULL, reps=1)
    assert not eng.factorize().any()
    eng.set_option('refine', 1)
    mean, var, _, _ = eng.predict(Z, Sigma, L.METHOD_TA)
    post = orc.postfit(X, Y, hyper, lapack_general_solve=False)
    mo, vo = orc.gp_mean_var(X, hyper, post['alpha'], post['chol'], Z)
    assert relinf(mean, mo) < 1e-6 and relinf(var, vo) < 1e-6
    eng.close()


@pytest.mark.parametrize('ctas', [1, 7, 133, 1000])
def test_half_tile_repeat_calls_are_bit_identical(ctas):
    eng, p = synthetic_engine(1100, 6, 8, seed=5, H=POOL)
    eng.set_option('predict_ctas', ctas)
    for H in (9, 56, 130):
        first = eng.predict(p['Z'][:H], p['Sigma'], L.METHOD_TA)
        again = eng.predict(p['Z'][:H], p['Sigma'], L.METHOD_TA)
        for x, y in zip(first, again):
            assert np.array_equal(x, y), H
        g1 = eng.predict_grad(p['Z'][:H], p['Sigma'], L.METHOD_TA)
        g2 = eng.predict_grad(p['Z'][:H], p['Sigma'], L.METHOD_TA)
        assert np.array_equal(g1['dvar_dz'], g2['dvar_dz']), H
    eng.close()

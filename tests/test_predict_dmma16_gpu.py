"""The predict product on DMMA.16x8x16: a point's var and cov do not depend on the chunk size (the BM instance of the
product kernel) or on the point's row in the chunk; var equals sf2 - |L^-1 ks|^2 formed from the engine's own L^-1;
repeat calls at a fixed stream-K partition are bit-identical."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._engines import synthetic_engine


pytestmark = pytest.mark.gpu

POOL = 130
HS = [1, 7, 8, 9, 50, 56, 64, 65, 130]


@pytest.mark.parametrize('Ny', [1, 8])
def test_point_results_do_not_depend_on_chunk_size_or_row(Ny):
    """N = 1000 (not a multiple of 128): the same points at shuffled rows of batches of every size give bitwise the
    same var and cov as in the full batch of 130 (two 64-point chunks and one of 2)."""
    eng, p = synthetic_engine(1000, 6, Ny, seed=4242 + Ny, H=POOL)
    Z, Sigma = p['Z'], p['Sigma']
    _, var_ref, cov_ref, _ = eng.predict(Z, Sigma, L.METHOD_TA)
    assert (var_ref > 0).all()
    rng = np.random.default_rng(Ny)
    for H in HS:
        for rep in range(2):
            idx = rng.permutation(POOL)[:H] if rep else (POOL - 1 - np.arange(H))
            _, var, cov, _ = eng.predict(Z[idx], Sigma, L.METHOD_TA)
            assert np.array_equal(var, var_ref[idx]), (H, rep)
            assert np.array_equal(cov, cov_ref[idx]), (H, rep)
    eng.close()


@pytest.mark.parametrize('Ny', [1, 8])
def test_var_matches_linv_ks_from_the_engine(Ny):
    """var = sf2 - |L^-1 ks|^2 with L^-1 read back from the engine (GET_LINV) and ks formed in numpy."""
    eng, p = synthetic_engine(1000, 6, Ny, seed=777 + Ny, H=POOL)
    X, Z, hyper = p['X'], p['Z'], p['hyper']
    Nx = X.shape[1]
    for H in (1, 50, 130):
        _, var, _, _ = eng.predict(Z[:H], None, L.METHOD_ME, want_cov=False, want_jac=False)
        for a in range(Ny):
            sf2 = hyper[a, Nx] ** 2
            ks = orc.covSEard(X, Z[:H], hyper[a, :Nx], sf2)             # (N, H)
            v = eng.get(L.GET_LINV, a) @ ks
            want = sf2 - np.einsum('nh,nh->h', v, v)
            # var = sf2 - |v|^2 cancels near the data: the rounding error scales with sf2, not with var
            assert np.abs(var[:, a] - want).max() < 1e-10 * sf2, (H, a)
    eng.close()


@pytest.mark.parametrize('ctas', [1, 7, 1000])
def test_repeat_calls_are_bit_identical(ctas):
    eng, p = synthetic_engine(1000, 6, 8, seed=99, H=POOL)
    eng.set_option('predict_ctas', ctas)
    for H in (9, 56, 130):
        first = eng.predict(p['Z'][:H], p['Sigma'], L.METHOD_TA)
        again = eng.predict(p['Z'][:H], p['Sigma'], L.METHOD_TA)
        for x, y in zip(first, again):
            assert np.array_equal(x, y), H
    eng.close()

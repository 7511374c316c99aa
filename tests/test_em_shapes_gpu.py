"""Exact moment matching ('EM', gpmpc_predict with METHOD_EM) against the long-double restatement of the reference's formula
(oracle gp_exact_moment(..., extended=True)) fed the engine's own alpha and a K^-1 from the engine's own Cholesky factor, at
every shape the EM kernels branch on:

* the register extent NXP of em_prep_kernel (8 / 16 / 32: Nx = 1, 8, 9, 12, 16, 17, 32; the Nx = 12 case runs in
  test_em_grad_gpu::test_em_forward_nxp16_vs_exact_moment);
* the 64-tiles of em_pair_kernel: mode 0 tiles ceil(N/64), mode 1 and the trace product Npad/64 (N = 1030: 17 vs 18);
* the feed of the lower-triangular trace product L^-1 Q~ (gemm128 with GEMM_KI_LE): 64x32 cp.async below 4 x SMs lower
  tiles, the TMA tensor-map kernel at Npad 3072;
* a reserved handle, whose identity tail of L^-1 enters the trace product;
* 45 and 990 output pairs (990 is the most em_finalize_kernel's 1024 threads allow, Ny = 44).

Every case runs at three input covariances: Sigma = 1e-5 Lambda (the remainder Q~ of Q_aa carries almost none of the
variance), 0.1 Lambda with a correlated off-diagonal part, and Lambda (the remainder carries a large share), with Lambda of
the output with the smallest length scales, and once as one per-point stack of all three.  The cross term cancels 4 to 6
digits, so errors are normalised by the sum of |terms| of each result (em_terms).  At Sigma >= 0.1 Lambda both parts of
the expected variance, the rank-one backbone t |L^-1 e^E|^2 and the remainder t tr(K^-1 Q~), must be at least 1e4 x the bar
x the normaliser, so losing or garbling either one fails the bar by orders of magnitude.  The measured errors quoted here
are from an H100 SXM (80 GB HBM3, 132 SMs) at its 700 W power limit."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._em_cases import (CASES, EM_TOL, SIGMAS, check_case, em_errors, em_terms, engine_factor, fit_case, sigmas,
                             tma_on_device)
from tests._engines import require

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', [n for n in CASES if n != 'nx12'])
def test_em_vs_long_double(name):
    """mean and cov of one-point calls and of a per-point stack of the three covariances against the reference.  Measured
    on an H100 SXM at 700 W, largest over the cases, the covariances and the two calls: mean 8.0e-17, cov 1.1e-16 (nx32
    at Sigma = Lambda, where the variance is all but sf2 and the normaliser is ~1) of the sums of |terms|; at sn = 1e-2
    mean 1.1e-17, cov 3.5e-19.  The smallest backbone or remainder at Sigma >= 0.1 Lambda is 5.0e-8 of its normaliser at
    sn = 0.3 (nx32 at Lambda) and 1.9e-10 at sn = 1e-2, against the guard's 1e4 x 1e-15.  var is diag(cov) and cov is
    symmetric bit for bit."""
    if name == 'tma':
        require(tma_on_device(), 'the TMA feed')
    check_case(name)


def test_em_points_are_independent_of_their_batch():
    """Each point gives the same bits alone, inside a per-point batch, inside a shared-Sigma batch and on a repeat call."""
    eng, X, Y, hyper, Z = fit_case('ny9')
    Sg = sigmas(hyper, X.shape[1])
    stack = np.stack([Sg[k] for k in SIGMAS])
    batch = eng.predict(Z, stack, L.METHOD_EM, want_jac=False)
    again = eng.predict(Z, stack, L.METHOD_EM, want_jac=False)
    shared = eng.predict(Z, Sg['0.1'], L.METHOD_EM, want_jac=False)
    for h, k in enumerate(SIGMAS):
        alone = eng.predict(Z[h:h + 1], Sg[k], L.METHOD_EM, want_jac=False)
        alone_shared = eng.predict(Z[h:h + 1], Sg['0.1'], L.METHOD_EM, want_jac=False)
        for i in range(3):
            assert np.array_equal(alone[i][0], batch[i][h]) and np.array_equal(batch[i][h], again[i][h]), (h, i)
            assert np.array_equal(alone_shared[i][0], shared[i][h]), (h, i)
    eng.close()


def test_em_scratch_shared_with_other_entry_points():
    """EM uses the handle's dKinv and dU as scratch, as GET_INVK, gpmpc_loo and gpmpc_predict_em_grad do (DESIGN 3): an EM
    prediction after those calls has the bits of one before them, and GET_INVK is unchanged by the EM calls."""
    eng, X, Y, hyper, Z = fit_case('nx8')
    Ny = Y.shape[1]
    S = sigmas(hyper, X.shape[1])['0.1']
    invk0 = [eng.get(L.GET_INVK, a) for a in range(Ny)]
    first = eng.predict(Z, S, L.METHOD_EM, want_jac=False)
    for a in range(Ny):
        eng.get(L.GET_INVK, a)
    eng.loo()
    eng.predict_em_grad(Z, S)
    second = eng.predict(Z, S, L.METHOD_EM, want_jac=False)
    for i in range(3):
        assert np.array_equal(first[i], second[i]), i
    for a in range(Ny):
        assert np.array_equal(eng.get(L.GET_INVK, a), invk0[a]), a
    eng.close()


@pytest.mark.parametrize('name', ['nx8', 'nx16'])
def test_em_cp_async_feeds_agree_bit_for_bit(name):
    """The trace product on 64x32 tiles (the default here, and small_tiles = 2^30) and on 128x64 tiles (small_tiles = 0)
    gives the same EM bits: both cp.async feeds sum each element's k-steps in the same order."""
    eng, X, Y, hyper, Z = fit_case(name)
    Sg = sigmas(hyper, X.shape[1])
    stack = np.stack([Sg[k] for k in SIGMAS])
    outs = []
    for st in (None, 0, 1 << 30):
        if st is not None:
            eng.set_option('small_tiles', st)
        outs.append(eng.predict(Z, stack, L.METHOD_EM, want_jac=False))
    for other in outs[1:]:
        for i in range(3):
            assert np.array_equal(outs[0][i], other[i]), i
    eng.close()


def tma_errors():
    """Npad 3072 at Sigma = Lambda: the errors of the trace product on the TMA feed and on 64x32 tiles (small_tiles = 2^30)
    against the reference, and of one against the other, under the reference's normalisation."""
    eng, X, Y, hyper, Z = fit_case('tma')
    alpha, kinv = engine_factor(eng, Y.shape[1])
    S = sigmas(hyper, X.shape[1])['1']
    ref = orc.gp_exact_moment(kinv, X, Y, hyper, Z[0], S, extended=True, beta=alpha)
    terms = em_terms(X, hyper, alpha, kinv, Z[0], S)
    tma = eng.predict(Z[:1], S, L.METHOD_EM, want_jac=False)
    eng.set_option('small_tiles', 1 << 30)
    cp = eng.predict(Z[:1], S, L.METHOD_EM, want_jac=False)
    eng.close()
    return dict(tma=em_errors(tma[0][0], tma[2][0], ref, terms), cp=em_errors(cp[0][0], cp[2][0], ref, terms),
                apart=em_errors(tma[0][0], tma[2][0], (cp[0][0], cp[2][0]), terms))


def test_em_tma_feed_agrees_with_cp_async():
    """At Npad 3072 the trace product on the TMA feed and on 64x32 tiles each meet the reference bar and agree with each
    other within it (the two sum the k-steps in different orders).  Measured on an H100 SXM at 700 W: TMA mean 2.2e-18,
    cov 9.1e-20, 64x32 mean 2.2e-18, cov 8.5e-20; apart: mean 0, cov 6.5e-21."""
    require(tma_on_device(), 'the TMA feed')
    tm, tc = EM_TOL
    for k, e in tma_errors().items():
        assert e['mean'] < tm and e['cov'] < tc, (k, e)


# (mean, var) bars of EM at Sigma = 1e-12 Lambda against ME: mean by the sum of |terms|, var by sf2
EM_ME_TOL = (2e-12, 2e-10)


def em_me_errors(name):
    """The largest errors of EM's mean (by sum_i |alpha_i k_i|) and variance (by sf2) at Sigma = 1e-12 Lambda against ME."""
    eng, X, Y, hyper, Z = fit_case(name)
    Nx, Ny = X.shape[1], Y.shape[1]
    S = 1e-12 * sigmas(hyper, Nx)['1']
    mean, var, _, _ = eng.predict(Z, S, L.METHOD_EM, want_jac=False)
    mean_me, var_me, _, _ = eng.predict(Z, None, L.METHOD_ME, want_jac=False)
    alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)])
    eng.close()
    sf2 = hyper[:, Nx] ** 2
    em = ev = 0.0
    for h in range(Z.shape[0]):
        ks = sf2[:, None] * np.exp(-0.5 * np.sum((X[None] - Z[h][None, None]) ** 2 / hyper[:, None, :Nx] ** 2, 2))
        em = max(em, np.max(np.abs(mean[h] - mean_me[h]) / np.abs(alpha * ks).sum(1)))
        ev = max(ev, np.max(np.abs(var[h] - var_me[h]) / sf2))
    return dict(mean=float(em), var=float(ev))


@pytest.mark.parametrize('name', ['nx8', 'nx32', 'tma'])
def test_em_tends_to_me(name):
    """As Sigma -> 0 the EM mean and variance tend to ME's: the backbone's variance is formed like ME's, so at
    Sigma = 1e-12 Lambda only the O(Sigma) terms separate them.  Measured on an H100 SXM at 700 W: mean <= 2.7e-13 of
    the sum of |terms|, var <= 5.2e-11 of sf2 (nx32; nx8 9.7e-15 / 2.8e-11, tma 4.4e-15 / 4.2e-11)."""
    if name == 'tma':
        require(tma_on_device(), 'the TMA feed')
    e = em_me_errors(name)
    assert e['mean'] < EM_ME_TOL[0] and e['var'] < EM_ME_TOL[1], e


def test_em_output_limit():
    """Ny = 44 (990 pairs) runs (case ny44 above); Ny = 45 is rejected with GPMPC_ERR_ARG and leaves the handle as it was:
    its next TA prediction has the bits of one made before the call."""
    import gp_mpc_b200
    N, Nx, Ny = 130, 3, 45
    p = orc.synthetic_problem(N, Nx, Ny, config_id=545, H=3)
    hyper = p['hyper'].copy()
    hyper[:, Nx + 1] = 0.3
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
    eng.set_data(p['X'], p['Y'])
    eng.set_hyper(hyper)
    assert not eng.factorize().any()
    S = 0.1 * np.eye(Nx)
    before = eng.predict(p['Z'], S, L.METHOD_TA)
    with pytest.raises(L.GpmpcError) as e:
        eng.predict(p['Z'], S, L.METHOD_EM, want_jac=False)
    assert e.value.code == L.ERR_ARG and 'Ny <= 44' in str(e.value)
    after = eng.predict(p['Z'], S, L.METHOD_TA)
    for x, y in zip(before, after):
        assert np.array_equal(x, y)
    eng.close()

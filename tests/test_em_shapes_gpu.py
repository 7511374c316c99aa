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
from scipy.linalg import cho_solve

from oracle import gp_oracle as orc
from tests.test_dispatch_gpu import _require, _sms, gemm_feed

pytestmark = pytest.mark.gpu

# name -> (N, Nx, Ny, capacity or None, sn)
CASES = {
    'nx1': (200, 1, 2, None, 0.3),          # NXP 8 with one live dimension; 200 mod 64 = 8
    'nx8': (1030, 8, 3, None, 0.3),         # top of the 8 bucket; T = 17, Tq = 18; Npad 1152 on 64x32
    'nx8_sn1e-2': (1030, 8, 3, None, 1e-2), # the same shape with cond(K) ~ 1e7
    'nx9': (700, 9, 2, None, 0.3),          # bottom of the 16 bucket
    'nx12': (600, 12, 3, None, 0.3),        # inside the 16 bucket (run by test_em_grad_gpu's forward Nx = 12 test)
    'nx16': (2150, 16, 2, None, 0.3),       # top of the 16 bucket; Npad 2176
    'nx17': (300, 17, 2, None, 0.3),        # NXP 32
    'nx32': (500, 32, 2, None, 0.3),        # NXP 32 full: em_pair's dynamic shared memory at its largest
    'tma': (3000, 6, 2, None, 0.3),         # Npad 3072: the trace product on the TMA feed
    'ny9': (400, 4, 9, None, 0.3),          # 45 pairs
    'ny44': (130, 3, 44, None, 0.3),        # 990 pairs, the limit
    'reserved': (1900, 6, 2, 2100, 0.3),    # Npad 2176 on a handle whose N would pad to 1920
}
SIGMAS = ('1e-5', '0.1', '1')
# (mean, cov) bars on the errors normalised by the sum of |terms|, for both conditionings: the reference takes the engine's
# alpha and factor, so cond(K) enters neither side's difference (measured maxima in test_em_vs_long_double)
EM_TOL = (1e-15, 1e-15)


def _L():
    import gp_mpc_b200
    return gp_mpc_b200._lib


def tma_on_device():
    """Npad 3072 puts the trace product's 24 x 25 lower tiles on the TMA feed (600 >= 4 x SMs up to 150 SMs)."""
    return gemm_feed(24, 24, 1, True, 1, _sms())[0] == 'tma'


def em_problem(name):
    """X, Y, hyper (sn of the case) and three test points of a case."""
    N, Nx, Ny, _, sn = CASES[name]
    p = orc.synthetic_problem(N, Nx, Ny, config_id=500 + Nx + Ny, H=3)
    hyper = p['hyper'].copy()
    hyper[:, Nx + 1] = sn
    return p['X'], p['Y'], hyper, p['Z']


def sigmas(hyper, Nx):
    """{'1e-5': 1e-5 Lambda, '0.1': 0.1 Lambda^1/2 (I + C) Lambda^1/2 / 2 with C a random correlation matrix, '1': Lambda},
    Lambda = diag(ell^2) of the output with the smallest length scales."""
    ell = hyper[np.argmin(np.sum(np.log(hyper[:, :Nx]), 1)), :Nx]
    A = np.random.default_rng(40 + Nx).standard_normal((Nx, Nx))
    M = A @ A.T
    d = np.sqrt(np.diag(M))
    corr = 0.5 * (np.eye(Nx) + M / np.outer(d, d))
    return {'1e-5': 1e-5 * np.diag(ell ** 2), '0.1': 0.1 * ell[:, None] * corr * ell[None, :], '1': np.diag(ell ** 2)}


def fit(name):
    import gp_mpc_b200
    N, Nx, Ny, cap, _ = CASES[name]
    X, Y, hyper, Z = em_problem(name)
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0, capacity=cap)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)
    assert not eng.factorize().any()
    return eng, X, Y, hyper, Z


def engine_factor(eng, Ny):
    """The engine's alpha (Ny, N) and K^-1 = cho_solve of its own Cholesky factor (Ny, N, N)."""
    L = _L()
    N = eng.N
    alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)])
    kinv = np.stack([cho_solve((eng.get(L.GET_CHOL, a), True), np.eye(N), check_finite=False) for a in range(Ny)])
    return alpha, 0.5 * (kinv + np.swapaxes(kinv, 1, 2))


def em_terms(X, hyper, beta, kinv, z, S):
    """Sums of |terms| of the EM moments at (z, S) and the two parts of the expected variance, in float64:
    mean_abs[a] = sum_i |beta_ai q_ai|; cov_abs[a, b] = sum_ij |beta_ai beta_bj tQ_ij|, plus sf2_a + sum_ij |K^-1_ij tQ_ij|
    when a = b; backbone[a] = t e^T K^-1 e and remainder[a] = t sum_ij K^-1_ij Q~_ij with Q_aa = e e^T + Q~."""
    Nx = X.shape[1]
    Ny = hyper.shape[0]
    v = X - z[None, :]
    ell2 = hyper[:, :Nx] ** 2
    sf2 = hyper[:, Nx] ** 2
    logk = [np.log(sf2[a]) - 0.5 * np.sum(v * v / ell2[a], 1) for a in range(Ny)]
    out = dict(mean_abs=np.zeros(Ny), cov_abs=np.zeros((Ny, Ny)), backbone=np.zeros(Ny), remainder=np.zeros(Ny))
    for a in range(Ny):
        R = S + np.diag(ell2[a])
        c = sf2[a] * np.prod(hyper[a, :Nx]) / np.sqrt(np.linalg.det(R))
        q = c * np.exp(-0.5 * np.sum((v @ np.linalg.inv(R)) * v, 1))
        out['mean_abs'][a] = np.abs(beta[a] * q).sum()
    for a in range(Ny):
        for b in range(a + 1):
            Rm = S @ np.diag(1.0 / ell2[a] + 1.0 / ell2[b]) + np.eye(Nx)
            t = 1.0 / np.sqrt(np.linalg.det(Rm))
            Qm = np.linalg.solve(Rm, 0.5 * S)
            ii = v / ell2[a]; ij = v / ell2[b]
            E = logk[a] + np.sum((ii @ Qm) * ii, 1)
            F = logk[b] + np.sum((ij @ Qm) * ij, 1)
            cr = 2.0 * (ii @ Qm) @ ij.T
            tQ = t * np.exp(E[:, None] + F[None, :] + cr)
            out['cov_abs'][a, b] = out['cov_abs'][b, a] = np.abs(beta[a]) @ tQ @ np.abs(beta[b])
            if a == b:
                e = np.exp(E)
                out['cov_abs'][a, a] += sf2[a] + np.abs(kinv[a] * tQ).sum()
                out['backbone'][a] = t * (e @ kinv[a] @ e)
                out['remainder'][a] = t * np.sum(kinv[a] * (np.outer(e, e) * np.expm1(cr)))
    return out


def em_errors(mean, cov, ref, terms):
    """Largest errors of one point's mean (Ny,) and cov (Ny, Ny) against ref = (mean, cov), normalised by terms."""
    return dict(mean=float(np.max(np.abs(mean - ref[0]) / terms['mean_abs'])),
                cov=float(np.max(np.abs(cov - ref[1]) / terms['cov_abs'])))


def check_bits(var, cov):
    """var is diag(cov) bit for bit and cov is exactly symmetric."""
    assert np.array_equal(var, np.einsum('haa->ha', cov))
    assert np.array_equal(cov, np.swapaxes(cov, 1, 2))


def case_errors(name):
    """Per input covariance: the errors of a one-point call and of the same point inside the per-point stack, and the
    smaller of backbone / remainder over the normaliser of its variance."""
    L = _L()
    _, Nx, Ny, _, _ = CASES[name]
    eng, X, Y, hyper, Z = fit(name)
    alpha, kinv = engine_factor(eng, Ny)
    Sg = sigmas(hyper, Nx)
    mean_s, var_s, cov_s, _ = eng.predict(Z, np.stack([Sg[k] for k in SIGMAS]), L.METHOD_EM, want_jac=False)
    check_bits(var_s, cov_s)
    out = {}
    for h, k in enumerate(SIGMAS):
        mean, var, cov, _ = eng.predict(Z[h:h + 1], Sg[k], L.METHOD_EM, want_jac=False)
        check_bits(var, cov)
        ref = orc.gp_exact_moment(kinv, X, Y, hyper, Z[h], Sg[k], extended=True, beta=alpha)
        terms = em_terms(X, hyper, alpha, kinv, Z[h], Sg[k])
        diag = np.diag(terms['cov_abs'])
        out[k] = dict(one=em_errors(mean[0], cov[0], ref, terms), stack=em_errors(mean_s[h], cov_s[h], ref, terms),
                      split=float(np.min(np.minimum(terms['backbone'], terms['remainder']) / diag)))
    eng.close()
    return out


def check_case(name):
    """Asserts the bars of case_errors(name) and, at Sigma >= 0.1 Lambda, that both parts of the expected variance are far
    above what the bar lets go missing."""
    tm, tc = EM_TOL
    for k, e in case_errors(name).items():
        for where in ('one', 'stack'):
            assert e[where]['mean'] < tm and e[where]['cov'] < tc, (name, k, where, e)
        if k != '1e-5':
            assert e['split'] >= 1e4 * tc, (name, k, e)


@pytest.mark.parametrize('name', [n for n in CASES if n != 'nx12'])
def test_em_vs_long_double(name):
    """mean and cov of one-point calls and of a per-point stack of the three covariances against the reference.  Measured
    on an H100 SXM at 700 W, largest over the cases, the covariances and the two calls: mean 8.0e-17, cov 1.1e-16 (nx32
    at Sigma = Lambda, where the variance is all but sf2 and the normaliser is ~1) of the sums of |terms|; at sn = 1e-2
    mean 1.1e-17, cov 3.5e-19.  The smallest backbone or remainder at Sigma >= 0.1 Lambda is 5.0e-8 of its normaliser at
    sn = 0.3 (nx32 at Lambda) and 1.9e-10 at sn = 1e-2, against the guard's 1e4 x 1e-15.  var is diag(cov) and cov is
    symmetric bit for bit."""
    if name == 'tma':
        _require(tma_on_device(), 'the TMA feed')
    check_case(name)


def test_em_points_are_independent_of_their_batch():
    """Each point gives the same bits alone, inside a per-point batch, inside a shared-Sigma batch and on a repeat call."""
    L = _L()
    eng, X, Y, hyper, Z = fit('ny9')
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
    L = _L()
    eng, X, Y, hyper, Z = fit('nx8')
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
    L = _L()
    eng, X, Y, hyper, Z = fit(name)
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
    L = _L()
    eng, X, Y, hyper, Z = fit('tma')
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
    _require(tma_on_device(), 'the TMA feed')
    tm, tc = EM_TOL
    for k, e in tma_errors().items():
        assert e['mean'] < tm and e['cov'] < tc, (k, e)


# (mean, var) bars of EM at Sigma = 1e-12 Lambda against ME: mean by the sum of |terms|, var by sf2
EM_ME_TOL = (2e-12, 2e-10)


def em_me_errors(name):
    """The largest errors of EM's mean (by sum_i |alpha_i k_i|) and variance (by sf2) at Sigma = 1e-12 Lambda against ME."""
    L = _L()
    eng, X, Y, hyper, Z = fit(name)
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
        _require(tma_on_device(), 'the TMA feed')
    e = em_me_errors(name)
    assert e['mean'] < EM_ME_TOL[0] and e['var'] < EM_ME_TOL[1], e


def test_em_output_limit():
    """Ny = 44 (990 pairs) runs (case ny44 above); Ny = 45 is rejected with GPMPC_ERR_ARG and leaves the handle as it was:
    its next TA prediction has the bits of one made before the call."""
    import gp_mpc_b200
    L = _L()
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

"""The 'EM' shape table of test_em_shapes_gpu (its module docstring says what each case reaches), the long-double checker
of one-point 'EM' moments, the cases of test_em_grad_gpu, and the feedback step of 'EM' roll-outs, shared by the 'EM'
prediction, derivative and roll-out tests on the device."""
import numpy as np
from scipy.linalg import cho_solve

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._engines import fit, gemm_feed, sms
from tests._util import load_fixture


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


def tma_on_device():
    """Npad 3072 puts the trace product's 24 x 25 lower tiles on the TMA feed (600 >= 4 x SMs up to 150 SMs)."""
    return gemm_feed(24, 24, 1, True, 1, sms())[0] == 'tma'


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


def fit_case(name):
    X, Y, hyper, Z = em_problem(name)
    eng, info = fit(X, Y, hyper, with_info=True, capacity=CASES[name][3])
    assert not info.any()
    return eng, X, Y, hyper, Z


def engine_factor(eng, Ny):
    """The engine's alpha (Ny, N) and K^-1 = cho_solve of its own Cholesky factor (Ny, N, N)."""
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
    _, Nx, Ny, _, _ = CASES[name]
    eng, X, Y, hyper, Z = fit_case(name)
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


def grad_case(case):
    """X, Y, hyper, Z, Sigma and the handle's capacity of a case; '<shape>_s<scale>' is a case of CASES at the
    input covariance of that scale (0.1 Lambda correlated, or Lambda)."""
    if '_s' in case:
        name, scale = case.split('_s')
        X, Y, hyper, Z = em_problem(name)
        return X, Y, hyper, Z[:1] if name == 'tma' else Z[:2], sigmas(hyper, X.shape[1])[scale], CASES[name][3]
    if case.startswith('tank'):
        m = load_fixture('tank'); X, Y, hyper = m['X'], m['Y'], m['hyper']
        rng = np.random.default_rng(5)
        Nx = X.shape[1]
        Z = X[rng.choice(X.shape[0], 4, replace=False)] + 0.05 * rng.standard_normal((4, Nx))
        A = rng.standard_normal((Nx, Nx)); Sigma = 1e-3 * np.eye(Nx) + 1e-4 * A @ A.T
        if case == 'tank_large':          # about a tenth of the smallest length scale squared
            Sigma = 0.1 * np.min(hyper[:, :Nx] ** 2) * (np.eye(Nx) + 0.1 * (A @ A.T) / np.abs(A @ A.T).max())
        if case == 'tank_pp':
            Sigma = np.stack([Sigma * (1 + 0.1 * h) for h in range(Z.shape[0])])
        return X, Y, hyper, Z, Sigma, None
    N, Nx, Ny, H = {'syn1000': (1000, 8, 4, 3), 'syn300': (300, 17, 2, 2), 'syn12': (600, 12, 3, 3)}[case]
    p = orc.synthetic_problem(N, Nx, Ny, config_id=N + Nx, H=H)
    hyper = p['hyper']
    if case == 'syn12':                   # well-conditioned (sn = 0.3): alpha and K^-1 carry no conditioning error
        hyper = hyper.copy(); hyper[:, Nx + 1] = 0.3
    return p['X'], p['Y'], hyper, p['Z'], p['Sigma'], None


def engine_alpha_chol(eng, Ny):
    """The engine's alpha (Ny, N) and Cholesky factor (Ny, N, N)."""
    return (np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)]),
            np.stack([eng.get(L.GET_CHOL, a) for a in range(Ny)]))


def feedback_sigma(S0, cov, K):
    """rollout_feedback_kernel's next Sigma from cov (Ny, Ny): sums in index order, no fused multiply-add."""
    Ny = cov.shape[0]
    S = S0.copy()
    S[:Ny, :Ny] = cov
    if K is None:
        return S
    Nu = K.shape[0]
    KC = np.zeros((Nu, Ny)); CK = np.zeros((Ny, Nu)); KCK = np.zeros((Nu, Nu))
    for k in range(Ny):
        KC = KC + K[:, k][:, None] * cov[k][None, :]
        CK = CK + cov[:, k][:, None] * K[:, k][None, :]
    for k in range(Ny):
        KCK = KCK + KC[:, k][:, None] * K[:, k][None, :]
    S[:Ny, Ny:] = CK; S[Ny:, :Ny] = CK.T; S[Ny:, Ny:] = KCK
    return S

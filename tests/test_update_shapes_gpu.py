"""The factor updates (gpmpc_remove, gpmpc_append, gpmpc_append_greedy) against the long-double restatement
oracle/update_oracle_ld.py applied to the engine's own pre-update factor, at every shape their kernels branch on:

* remove_coef_kernel's rows per thread (m up to 2049: 1, 2 and 3 rows), remove_l_rows_kernel's carry across its
  256-element segments (m = 255 / 256 / 257 / 513 / 1024 / 1025 / 2049), the RM_RB = 64 row blocks of remove_li_part /
  _scan / _apply (m = 63 / 64 / 65 / 128, row blocks in which the diagonal 128-block changes), indices 0, 127, 128,
  129, N - 2 and N - 1 (m = 0: the commit and the shift alone), 129 -> 128 points, N = Npad with no spare row, several
  indices in one call (adjacent and across blocks), three outputs and a sharded handle (out_begin = 1);
* append_row_kernel onto N = 127 and 128 of a reserved handle (the new row last in its 128-block, first in a fresh
  one), N + 1 = Npad, Nx = 1 and 32 with 8 outputs, and a near-duplicate point (lambda^2 ~ 1e-6 sf2);
* greedy_pick_kernel over pools of 1025 and 2100 candidates (more than its 1024 threads), exact ties of duplicated
  candidates, Ny = 40 (its second round of Y stores), Nx = 1 and 32, greedy_downdate_kernel with Nk crossing a
  128-boundary and reaching Npad;
* an append onto a factor that needed the jitter retry, and 2048 cycles of a sliding window at N = Npad = 1024.

Each updated row of L and L^-1 (every row from the first removed index on for a removal; the rows above must keep
their bits), alpha and log det are compared with the reference, normalised entry by entry by the reference's sum of
|terms|.  GET_CHOL and GET_LINV show only the N x N lower triangle, so each case then predicts (TA) at points next to
the edited rows: the predict product also reads the upper triangle of each diagonal 128-block and the identity tail
rows >= N, and a stale value left there changes var, which is compared with the long-double reference on the
engine's post-update alpha and L^-1 with the normalisation and bars of test_predict_derivs_shapes_gpu.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, largest normalised error over every case (case in
brackets):

    L 2.5e-16 (ny40)   L^-1 3.0e-16 (m2049)   alpha 1.6e-16 (m1)   log det 1.2e-16 (m1025)   greedy score 1.2e-17 (nx32)
    predict after the update: mean 1.1e-16, var 6.6e-17, J 2.3e-16, cov 5.6e-17 (all nx32_ny8)

and on the jittered factor no larger (L 1.9e-16, L^-1 1.5e-16).  TOL is 10x each maximum rounded up in its first
digit; the predict bars are test_predict_derivs_shapes_gpu's.  The window's drift after 256 / 2048 cycles: backward
error 2.8e-14 / 1.1e-13, max|L^-1 L - I| 2.7e-14 / 4.3e-14, against 3.6e-15 / 1.6e-14 for the fresh factorisation of
the first window; DRIFT_TOL is about 10x the larger of each."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import hess_oracle as hor
from oracle import update_oracle_ld as upd
from tests._util import PREDICT_TOL, normalised

pytestmark = pytest.mark.gpu

LD = np.longdouble
# bars on the largest error normalised by the sum of |terms| (measured maxima in the module docstring)
TOL = dict(L=3e-15, Li=4e-15, alpha=2e-15, logdet=2e-15, score=2e-16)
PRED = ('mean', 'var', 'jac', 'cov')
REF_KEY = dict(jac='J')
# the sliding window: backward error max|L L^T - K| / max|K| and max|L^-1 L - I| after 256 and 2048 cycles
DRIFT_TOL = dict(backward=1e-12, inverse=4e-13)


def problem(N, Nx, Ny, sn=0.3, seed=0):
    p = orc.synthetic_problem(N, Nx, Ny, config_id=900 + 7 * Nx + Ny + seed)
    hyper = p['hyper'].copy()
    hyper[:, Nx + 1] = sn
    return p['X'], p['Y'], hyper


def fit(X, Y, hyper, cap=None, out_begin=0, out_count=None):
    eng = L.Engine(X.shape[0], X.shape[1], Y.shape[1], device=0, capacity=cap, out_begin=out_begin,
                      out_count=out_count)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)
    info = eng.factorize()
    return eng, info


def factors(eng):
    return [upd.factor(eng.get(L.GET_CHOL, a), eng.get(L.GET_LINV, a)) for a in eng.local_outputs]


def worst(x, ref, scale):
    """Largest |x - ref| / scale; an entry whose scale is 0 must be 0 on both sides."""
    return normalised(np.asarray(x), np.asarray(ref, dtype=LD), np.asarray(scale, dtype=LD))


def check(eng, pre, post, rows, X, Y, hyper, near):
    """The engine after an update against the reference Factors `post` (one per owned output): rows < rows keep the
    bits of `pre`, rows >= rows within the scales; alpha and log det; then TA at H = 8 points 0.05 from the training
    inputs `near` (skipped on a sharded handle).  X, Y: the data after the update; hyper: the owned rows.
    Returns the largest normalised error of each quantity."""
    got = factors(eng)
    N = X.shape[0]
    err = dict(L=0.0, Li=0.0, alpha=0.0, logdet=0.0)
    for a, (g, F, P) in enumerate(zip(got, post, pre)):
        assert g.L.shape == (N, N)
        r0 = min(rows, P.L.shape[0])
        assert np.array_equal(g.L[:r0, :r0], P.L[:r0, :r0]) and np.array_equal(g.Li[:r0, :r0], P.Li[:r0, :r0])
        err['L'] = max(err['L'], worst(g.L[rows:], F.L[rows:], F.SL[rows:]))
        err['Li'] = max(err['Li'], worst(g.Li[rows:], F.Li[rows:], F.SLi[rows:]))
        ga = eng.get(L.GET_ALPHA, eng.out_begin + a)
        ra, sa = upd.alpha(F, Y[:, eng.out_begin + a])
        err['alpha'] = max(err['alpha'], worst(ga, ra, sa))
        gl = eng.get(L.GET_LOGDET, eng.out_begin + a)[0]
        rl, sl = upd.logdet(F)
        err['logdet'] = max(err['logdet'], float(abs(LD(gl) - rl) / sl))
    if eng.out_begin == 0 and eng.out_count == eng.Ny:
        Nx = X.shape[1]
        rng = np.random.default_rng(N)
        sel = np.round(np.linspace(0, len(near) - 1, 8)).astype(int)
        Z = np.asarray(near)[sel] + 0.05 * rng.standard_normal((8, Nx))
        S = 0.01 * np.diag(np.mean(hyper[:, :Nx], 0) ** 2)
        m, v, c, J = eng.predict(Z, S, L.METHOD_TA)
        out = dict(mean=m, var=v, cov=c, jac=J)
        alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(eng.Ny)])
        linv = np.stack([x.Li for x in got])
        ref = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, 'TA')
        ab = hor.predict_derivs_ld(X, hyper, alpha, linv, Z, S, 'TA', absolute=True)
        for k in PRED:
            err[k] = normalised(out[k], ref[REF_KEY.get(k, k)], ab[REF_KEY.get(k, k)])
    return err


def assert_within(name, err):
    print('MEASURED', name, {k: '%.2e' % v for k, v in err.items()})
    bad = {k: e for k, e in err.items() if not e <= TOL.get(k, PREDICT_TOL.get(k))}
    assert not bad, (name, bad)


# ----------------------------------------------------------------------------------------------------- removal
# name -> (N, Nx, Ny, indices, out_begin)
REMOVE = {
    'i0': (300, 4, 2, [0], 0),
    'i127': (300, 4, 2, [127], 0),
    'i128': (300, 4, 2, [128], 0),
    'i129': (300, 4, 2, [129], 0),
    'iNm2': (300, 4, 2, [298], 0),
    'iNm1_m0': (300, 4, 2, [299], 0),                 # the last point: only the commit and the shift run
    'm1': (700, 3, 1, [698], 0),
    'm63': (700, 3, 1, [636], 0),                      # one partial row block; rows 636 .. 698 cross 640
    'm64': (700, 3, 1, [635], 0),
    'm65': (700, 3, 1, [634], 0),                      # a second row block of one row
    'm128': (700, 3, 1, [571], 0),
    'm255': (700, 3, 1, [444], 0),
    'm256': (700, 3, 1, [443], 0),
    'm257': (700, 3, 1, [442], 0),                     # the L rows' second 256-element segment
    'm513': (2100, 3, 1, [1586], 0),                   # three segments; coef: one row per thread
    'm1024': (2100, 3, 1, [1075], 0),
    'm1025': (2100, 3, 1, [1074], 0),                  # coef: two rows per thread
    'm2049': (2100, 3, 1, [50], 0),                    # coef: three rows per thread; nine segments
    '129to128': (129, 4, 2, [5], 0),
    'full_pad': (1024, 4, 1, [300], 0),                # N = Npad: the freed row is the slab's last
    'adjacent': (700, 3, 2, [200, 201, 202], 0),
    'across_blocks': (700, 3, 2, [5, 127, 128, 400, 699], 0),
    'ny3': (500, 4, 3, [130, 7], 0),
    'sharded': (500, 4, 3, [250, 3], 1),               # outputs 1 and 2 of 3
}


@pytest.mark.parametrize('name', list(REMOVE))
def test_remove_vs_long_double(name):
    """Every row of L and L^-1 from the first removed index on, alpha and log det after gpmpc_remove, then TA next to
    the moved rows, against the reference on the engine's pre-removal factor."""
    N, Nx, Ny, idx, ob = REMOVE[name]
    X, Y, hyper = problem(N, Nx, Ny)
    eng, info = fit(X, Y, hyper, out_begin=ob, out_count=Ny - ob)
    assert not info.any()
    pre = factors(eng)
    post = [upd.remove(F, idx) for F in pre]
    eng.remove(idx)
    keep = np.setdiff1d(np.arange(N), idx)
    Xk = X[keep]
    i0 = min(idx)
    near = np.vstack([Xk[max(i0 - 1, 0):], X[idx]])     # the moved rows and the removed points' neighbourhoods
    err = check(eng, pre, post, i0, Xk, Y[keep], hyper[ob:], near)
    eng.close()
    assert_within(name, err)


# ------------------------------------------------------------------------------------------------------ append
# name -> (N, Nx, Ny, capacity, sn)
APPEND = {
    'n127_to_128': (127, 4, 2, 300, 0.3),              # the new row is the last of block 0 (Npad 384)
    'n128_to_129': (128, 4, 2, 300, 0.3),              # the new row opens block 1 of a reserved handle
    'fill_npad': (255, 4, 2, None, 0.3),               # N + 1 = Npad
    'nx1_ny8': (400, 1, 8, 500, 0.3),
    'nx32_ny8': (400, 32, 8, 500, 0.3),
    'near_duplicate': (300, 4, 1, None, 7e-4),         # lambda^2 ~ 1e-6 sf2
}


@pytest.mark.parametrize('name', list(APPEND))
def test_append_vs_long_double(name):
    """Row N of L and L^-1 after gpmpc_append (rows < N keep their bits), alpha and log det, then TA next to the new
    point, against the reference on the engine's pre-append factor."""
    N, Nx, Ny, cap, sn = APPEND[name]
    X, Y, hyper = problem(N + 1, Nx, Ny, sn=sn)
    x_new, y_new = X[N], Y[N]
    if name == 'near_duplicate':
        x_new = X[N // 2].copy()
    X, Y = X[:N], Y[:N]
    eng, info = fit(X, Y, hyper, cap=cap)
    assert not info.any()
    pre = factors(eng)
    res = [upd.append_point(F, X, x_new, hyper[a]) for a, F in enumerate(pre)]
    if name == 'near_duplicate':
        lam2 = float(res[0][1] ** 2) / hyper[0, Nx] ** 2
        assert 1e-7 < lam2 < 1e-5, lam2
    assert eng.append(x_new, y_new)
    Xn, Yn = np.vstack([X, x_new]), np.vstack([Y, y_new])
    err = check(eng, pre, [r[0] for r in res], N, Xn, Yn, hyper, np.vstack([x_new, X[-4:]]))
    eng.close()
    assert_within(name, err)


def test_append_onto_a_jittered_factor():
    """Output 1 of 3 has duplicated points and sn = 1e-10, so gpmpc_factorize needs its jitter retry (info [0, 1, 0])
    and holds the factor of K + 1e-8 I.  A far point and then a near one are appended, with a K build in between
    (GET_K, which reuses the K build's jitter scratch).  Each new row must be the factor of K_aug + 1e-8 I: the
    reference puts the jitter on the new diagonal entry of output 1 and on none of the others."""
    N, Nx = 300, 6
    X, Y, hyper = problem(N + 2, Nx, 3, sn=1e-2, seed=1)
    X[N // 2:N] = X[:N - N // 2]
    hyper[1, Nx + 1] = 1e-10
    jit = np.array([0.0, 1e-8, 0.0])
    eng, info = fit(X[:N], Y[:N], hyper)
    assert list(info) == [0, 1, 0]
    pts = [X[0] + 3.0, X[7] + 1e-3]
    Xc, Yc = X[:N], Y[:N]
    errs = {}
    for step, x in enumerate(pts):
        eng.get(L.GET_K, 1)
        pre = factors(eng)
        res = [upd.append_point(F, Xc, x, hyper[a], jitter=jit[a]) for a, F in enumerate(pre)]
        assert eng.append(x, Y[N + step])
        Xc, Yc = np.vstack([Xc, x]), np.vstack([Yc, Y[N + step]])
        err = check(eng, pre, [r[0] for r in res], Xc.shape[0] - 1, Xc, Yc, hyper, np.vstack([x, Xc[:8]]))
        errs.update({'%s %d' % (k, step): v for k, v in err.items()})
    # the jittered output's new diagonal: (l^T l + lambda^2) = sf2 + sn2 + 1e-8 to rounding
    Lg = eng.get(L.GET_CHOL, 1).astype(LD)
    kd = LD(hyper[1, Nx]) ** 2 + LD(hyper[1, Nx + 1]) ** 2 + LD(1e-8)
    assert abs(float(Lg[-1] @ Lg[-1] - kd)) < 1e-14
    eng.close()
    print('MEASURED jitter', {k: '%.2e' % v for k, v in errs.items()})
    bad = {k: e for k, e in errs.items() if not e <= TOL.get(k.split()[0], PREDICT_TOL.get(k.split()[0]))}
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------ greedy
# name -> (N, Nx, Ny, capacity, pool size, n_new, duplicated pool)
GREEDY = {
    'pool1025': (300, 4, 2, 320, 1025, 3, False),
    'pool2100': (300, 4, 2, 320, 2100, 2, False),
    'ties': (300, 4, 2, 320, 200, 4, True),            # every candidate twice: the lower index wins
    'ny40': (200, 3, 40, None, 300, 3, False),
    'nx1': (200, 1, 2, None, 300, 3, False),
    'nx32': (200, 32, 2, None, 300, 3, False),
    'across_128': (120, 4, 2, 256, 300, 12, False),    # Nk = 120 .. 131
    'to_npad': (240, 4, 2, None, 300, 16, False),      # Nk = 240 .. 255: the last row of the slab
}


@pytest.mark.parametrize('name', list(GREEDY))
def test_greedy_vs_long_double(name):
    """The picks (equal; each pick stands clear of every distinct candidate's score by 1e4 x the score's bar, so the
    comparison is not decided by rounding), their scores, the new rows of L and L^-1, alpha and log det after
    gpmpc_append_greedy, then TA next to the picked points, against the reference on the pre-selection factor."""
    N, Nx, Ny, cap, n, n_new, dup = GREEDY[name]
    X, Y, hyper = problem(N + n, Nx, Ny)
    Xc, Yc = X[N:], Y[N:]
    if dup:
        Xc[n // 2:], Yc[n // 2:] = Xc[:n // 2], Yc[:n // 2]
    X, Y = X[:N], Y[:N]
    eng, info = fit(X, Y, hyper, cap=cap)
    assert not info.any()
    pre = factors(eng)
    ref = upd.greedy(pre, X, hyper, Xc, n_new)
    assert np.all(ref['gap'] > 1e4 * TOL['score']), ref['gap']
    picked, score, ok = eng.append_greedy(Xc, Yc, n_new)
    assert ok and list(picked) == list(ref['picked'])
    if dup:
        assert picked[0] < n // 2
    Xn, Yn = np.vstack([X, Xc[picked]]), np.vstack([Y, Yc[picked]])
    err = check(eng, pre, ref['Fs'], N, Xn, Yn, hyper, Xc[picked])
    err['score'] = worst(score, ref['score'], ref['sscore'])
    eng.close()
    assert_within(name, err)


# ------------------------------------------------------------------------------------------------------- drift
def drift(L, Li, X, hyper_a):
    """(max|L L^T - K| / max|K|, max|L^-1 L - I|) in long double, K by direct differences of the window X."""
    L, Li = np.asarray(L, dtype=LD), np.asarray(Li, dtype=LD)
    K = upd.kvec(X, X, hyper_a) + LD(hyper_a[-1]) ** 2 * np.eye(X.shape[0], dtype=LD)
    be = float(np.max(np.abs(L @ L.T - K)) / np.max(np.abs(K)))
    ie = float(np.max(np.abs(Li @ L - np.eye(X.shape[0], dtype=LD))))
    return be, ie


def test_sliding_window_drift():
    """A window of N = Npad = 1024 points (no spare row) slides through 2048 cycles of remove([0]) + append; after 256
    and 2048 cycles the factor's backward error against the window's K and the error of L^-1 as L's inverse stay
    within DRIFT_TOL (compare the fresh factorisation's, printed alongside)."""
    N, Nx, C = 1024, 4, 2048
    X, Y, hyper = problem(N + C, Nx, 1, sn=0.1)
    eng, info = fit(X[:N], Y[:N], hyper)
    assert not info.any() and eng.capacity == N
    got = {0: drift(eng.get(L.GET_CHOL, 0), eng.get(L.GET_LINV, 0), X[:N], hyper[0])}
    for c in range(1, C + 1):
        eng.remove([0])
        assert eng.append(X[N + c - 1], Y[N + c - 1])
        if c in (256, C):
            got[c] = drift(eng.get(L.GET_CHOL, 0), eng.get(L.GET_LINV, 0), X[c:N + c], hyper[0])
    eng.close()
    print('MEASURED drift', {c: ('%.2e' % b, '%.2e' % i) for c, (b, i) in got.items()})
    for c in (256, C):
        assert got[c][0] <= DRIFT_TOL['backward'] and got[c][1] <= DRIFT_TOL['inverse'], got

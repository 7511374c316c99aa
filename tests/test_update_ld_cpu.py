"""oracle/update_oracle_ld.py (the long-double restatement of gpmpc_append, gpmpc_append_greedy and gpmpc_remove that
tests/test_update_shapes_gpu.py measures the kernels against) on the CPU: against the same formulas in 40-digit
mpmath, against the float64 remove_oracle and greedy_oracle, and against the matrix it must factorise."""
import mpmath as mp
import numpy as np
import pytest

from oracle import gp_oracle as orc
from oracle import greedy_oracle as gro
from oracle import remove_oracle as rmo
from oracle import update_oracle_ld as upd

LD = np.longdouble


def problem(N, Nx=3, Ny=1, seed=0, sn=0.3):
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((N, Nx))
    hyper = np.zeros((Ny, Nx + 2))
    hyper[:, :Nx] = rng.uniform(0.8, 2.0, (Ny, Nx))
    hyper[:, Nx] = rng.uniform(0.8, 1.5, Ny)
    hyper[:, Nx + 1] = sn
    return X, hyper


def K_ld(X, hyper_a, jitter=0.0):
    """K + (sn2 + jitter) I by direct differences, in long double."""
    return upd.kvec(X, X, hyper_a) + (LD(hyper_a[-1]) ** 2 + LD(jitter)) * np.eye(X.shape[0], dtype=LD)


def engine_like(X, hyper_a):
    """A float64 (L, L^-1) pair as an engine would hold it: LAPACK's factor and its triangular inverse."""
    L = np.linalg.cholesky(orc.assemble_K(X, hyper_a))
    return L, np.linalg.inv(L)


def accurate_pair(K):
    """L and L^-1 of K (long double) to long-double accuracy: 40-digit Cholesky and inverse, rounded."""
    with mp.workdps(40):
        Lm = mp.cholesky(mp.matrix([[mp.mpf(str(v)) for v in row] for row in K]))
        Lim = Lm ** -1
        n = K.shape[0]
        to = lambda M: np.array([[LD(mp.nstr(M[r, c], 30)) for c in range(n)] for r in range(n)], dtype=LD)
        return to(Lm), to(Lim)


def mpm(A):
    if isinstance(A, mp.matrix):
        return A
    return mp.matrix([[mp.mpf(float(v)) for v in row] for row in np.asarray(A, dtype=np.float64)])


def worst(x, ref, scale):
    """Largest |x - ref| / scale (ref an mpmath matrix)."""
    e = 0.0
    for r in range(x.shape[0]):
        for c in range(x.shape[1]):
            d = abs(mp.mpf(str(x[r, c])) - ref[r, c])
            if d:
                assert scale[r, c] > 0, (r, c)
                e = max(e, float(d / mp.mpf(str(scale[r, c]))))
    return e


def mp_append(L, Li, k, kss):
    """The append in 40 digits: row N of L and of L^-1 (1 x (N+1) each)."""
    L, Li, k = mpm(L), mpm(Li), mp.matrix([mp.mpf(str(v)) for v in k])
    N = L.rows
    l = Li * k
    lam = mp.sqrt(mp.mpf(str(kss)) - sum(l[j] ** 2 for j in range(N)))
    rl, rli = mp.matrix(1, N + 1), mp.matrix(1, N + 1)
    for j in range(N):
        rl[0, j] = l[j]
        rli[0, j] = -sum(l[q] * Li[q, j] for q in range(N)) / lam
    rl[0, N], rli[0, N] = lam, 1 / lam
    return rl, rli


def mp_remove(L, Li, i):
    """The removal of point i in 40 digits, by the kernels' formulas written as plain loops."""
    L, Li = mpm(L), mpm(Li)
    N = L.rows
    keep = [c for c in range(N) if c != i]
    n = N - i - 1
    p = [-L[i, i] * Li[i + 1 + r, i] for r in range(n)]
    t, tp = [], mp.mpf(1)
    d, g = [], []
    for r in range(n):
        tr = tp + p[r] ** 2
        d.append(mp.sqrt(tr / tp))
        g.append(p[r] / mp.sqrt(tr * tp))
        tp = tr
    L2 = mp.matrix(N - 1, N - 1)
    Li2 = mp.matrix(N - 1, N - 1)
    for r, R in enumerate(keep):
        for c, C in enumerate(keep):
            L2[r, c], Li2[r, c] = L[R, C], Li[R, C]
    Rm = [[Li[i + 1 + r, C] + p[r] * Li[i, C] for C in keep] for r in range(n)]
    for r in range(n):
        for c in range(i):
            L2[i + r, c] = L[i + 1 + r, c]
        for j in range(r + 1):
            s = sum(p[k] * L[i + 1 + r, i + 1 + k] for k in range(j + 1, r + 1))
            L2[i + r, i + j] = d[j] * L[i + 1 + r, i + 1 + j] + g[j] * s
        for c in range(N - 1):
            s = sum(p[q] * Rm[q][c] for q in range(r))
            Li2[i + r, c] = Rm[r][c] / d[r] - g[r] * s
    return L2, Li2


@pytest.mark.parametrize('N', [1, 9, 14])
def test_append_vs_mpmath(N):
    """Row N of both factors within 1e-17 of the sums of |terms| of the same formulas in 40 digits; rows < N as given."""
    X, hyper = problem(N + 1, seed=N)
    L, Li = engine_like(X[:N], hyper[0])
    F, lam, slam = upd.append_point(upd.factor(L, Li), X[:N], X[N], hyper[0])
    k = upd.kvec(X[:N], X[N], hyper[0])[:, 0]
    with mp.workdps(40):
        rl, rli = mp_append(L, Li, k, upd.kss(hyper[0]))
        assert worst(F.L[N:], rl, F.SL[N:]) < 1e-17
        assert worst(F.Li[N:], rli, F.SLi[N:]) < 1e-17
    assert np.array_equal(F.L[:N, :N], L) and np.array_equal(F.Li[:N, :N], Li)
    assert not F.L[:N, N].any() and not F.Li[:N, N].any()
    assert lam == F.L[N, N] and slam >= lam


@pytest.mark.parametrize('N,idx', [(12, [0]), (12, [5]), (12, [10]), (12, [11]), (13, [2, 7, 12]), (13, [4, 5, 6])])
def test_remove_vs_mpmath(N, idx):
    """Every entry of both factors within 1e-17 of its scale of the kernels' formulas in 40 digits (several indices:
    one at a time in descending order, each on the previous 40-digit result)."""
    X, hyper = problem(N, seed=N + len(idx))
    L, Li = engine_like(X, hyper[0])
    F = upd.remove(upd.factor(L, Li), idx)
    with mp.workdps(40):
        Lm, Lim = L, Li
        for i in sorted(idx, reverse=True):
            Lm, Lim = mp_remove(Lm, Lim, i)
        assert worst(F.L, Lm, F.SL) < 1e-17
        assert worst(F.Li, Lim, F.SLi) < 1e-17


@pytest.mark.parametrize('N,idx', [(40, [0]), (40, [17]), (40, [39]), (41, [3, 20, 40])])
def test_remove_vs_float64_oracle(N, idx):
    """The float64 remove_oracle (a different vectorisation of the same formulas) agrees to 1e-14 of the scales."""
    X, hyper = problem(N, seed=3)
    L, Li = engine_like(X, hyper[0])
    F = upd.remove(upd.factor(L, Li), idx)
    L2, Li2 = rmo.remove(L, Li, idx)
    for x, ref, s in ((F.L, L2, F.SL), (F.Li, Li2, F.SLi)):
        d = np.abs(np.asarray(x, dtype=np.float64) - ref)
        assert np.all(d <= 1e-14 * np.asarray(s, dtype=np.float64)), float(np.max(d / np.where(s > 0, s, 1)))


@pytest.mark.parametrize('op', ['append', 'remove_first', 'remove_middle', 'remove_several', 'greedy'])
def test_updated_factor_reproduces_the_new_K(op):
    """From a long-double-accurate pair of K, each update leaves L' with L' L'^T = K' to long-double precision (K' the
    direct-difference K of the new data), L^-1' L' = I likewise, and alpha / log det of the new data."""
    N = 30
    X, hyper = problem(N + 40, seed=11)
    h = hyper[0]
    L, Li = accurate_pair(K_ld(X[:N], h))
    F = upd.Factor(L, Li, np.abs(L), np.abs(Li))
    if op == 'append':
        F, _, _ = upd.append_point(F, X[:N], X[N], h)
        Xn = X[:N + 1]
    elif op == 'greedy':
        out = upd.greedy([F], X[:N], hyper, X[N:], 5)
        F = out['Fs'][0]
        Xn = np.vstack([X[:N], X[N:][out['picked']]])
    else:
        idx = {'remove_first': [0], 'remove_middle': [13], 'remove_several': [2, 3, 17, 29]}[op]
        F = upd.remove(F, idx)
        Xn = np.delete(X[:N], idx, axis=0)
    K = K_ld(Xn, h)
    n = Xn.shape[0]
    assert F.L.shape == (n, n)
    assert float(np.max(np.abs(F.L @ F.L.T - K)) / np.max(np.abs(K))) < 1e-17
    assert float(np.max(np.abs(F.Li @ F.L - np.eye(n, dtype=LD)))) < 1e-16
    assert not np.triu(F.L, 1).any() and not np.triu(F.Li, 1).any()
    y = np.sin(np.arange(n, dtype=np.float64))
    a, sa = upd.alpha(F, y)
    assert float(np.max(np.abs(K @ a - y))) < 1e-16 and np.all(sa >= np.abs(a))
    ld_, sld = upd.logdet(F)
    assert abs(float(ld_) - np.linalg.slogdet(np.asarray(K, dtype=np.float64))[1]) < 1e-12 and sld >= abs(ld_)


def test_jitter_enters_the_new_diagonal():
    """append_point with the output's jitter j factorises K_aug + j I: the new diagonal of L' L'^T is kss + j."""
    N, j = 20, 1e-6
    X, hyper = problem(N + 1, seed=5)
    h = hyper[0]
    L, Li = accurate_pair(K_ld(X[:N], h, j))
    F, _, _ = upd.append_point(upd.Factor(L, Li, np.abs(L), np.abs(Li)), X[:N], X[N], h, jitter=j)
    K = K_ld(X[:N + 1], h, j)
    assert float(np.max(np.abs(F.L @ F.L.T - K))) < 1e-17


def test_scales_bound_their_entries():
    """Every sum of |terms| is at least |its entry| after each kind of update."""
    X, hyper = problem(60, Ny=2, seed=9)
    for a in range(2):
        L, Li = engine_like(X[:40], hyper[a])
        F0 = upd.factor(L, Li)
        for F in (upd.append_point(F0, X[:40], X[40], hyper[a])[0], upd.remove(F0, [0, 7, 39])):
            assert np.all(F.SL >= np.abs(F.L)) and np.all(F.SLi >= np.abs(F.Li))


@pytest.mark.parametrize('dup', [False, True])
def test_greedy_picks_match_greedy_oracle(dup):
    """Picks and order equal the float64 greedy_oracle (a refit per step, no downdates), scores within 1e-10 of it,
    with a pool holding every candidate twice: the lowest index of equal scores wins, as on the device.  The updated
    factors equal those of appending the picked points one by one (l = L^-1 k instead of the downdated V) to 1e-17 of
    their scales."""
    X, hyper = problem(30 + 25, Nx=2, Ny=2, seed=21)
    Xt, Xc = X[:30], X[30:]
    if dup:
        Xc = np.vstack([Xc, Xc])
    Fs = [upd.factor(*engine_like(Xt, hyper[a])) for a in range(2)]
    out = upd.greedy(Fs, Xt, hyper, Xc, 6)
    ref = gro.greedy_select(Xt, hyper, Xc, 6)
    assert list(out['picked']) == list(ref['picked'])
    assert out['picked'][0] < 25                     # every score has its twin at the first pick
    assert np.max(np.abs(np.asarray(out['score'], dtype=np.float64) - ref['score'])) < 1e-10
    Xg = Xt
    for a in range(2):
        F, Xg = Fs[a], Xt
        for c in out['picked']:
            F, _, _ = upd.append_point(F, Xg, Xc[c], hyper[a])
            Xg = np.vstack([Xg, Xc[c]])
        G = out['Fs'][a]
        for x, ref_, s in ((G.L, F.L, G.SL), (G.Li, F.Li, G.SLi)):
            assert float(np.max(np.abs(x - ref_) / np.where(s > 0, s, 1))) < 1e-17

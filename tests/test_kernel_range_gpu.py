"""Every kernel value the engine computes, sf2 exp(-1/2 |(x - z)/ell|^2) = 2^t, across the whole range of t the fit's
bounds reach (ell down to 1e-2 on standardised data puts t far below the clamp at -1020), entry by entry against a
long-double direct-difference reference, never against the engine's own K:

B1. the full K build (gpmpc_build_K) on 1-D grids and Nx = 8, 17, 32 designs with sf in {2^-20, 1, 2^6 3}: every entry
    within its own bound (tests/_kernel_range.py) relative to its own magnitude, entries whose exact t is below the
    clamp equal to 2^-1020 bit for bit, the diagonal, and exact duplicates in different 128-tiles;
B2. the lower build the factorisation uses, in its checked and unchecked bodies, through L: on designs whose
    off-diagonal entries are all below 2^-30 sf2, L_ij L_jj = K_ij to rounding;
B3. every ks value through gpmpc_predict with training points so far apart that K is diagonal and one-hot targets, so
    mean and J are single terms, for every ks chunk CH with the NXP values it pairs with;
B4. six regimes end to end (short ell, long ell with sn/sf = 1e-5, ARD from 1e-2 to 1e4, sf = 3 2^+-10 with
    sn/sf in {1e-5, 0.5}, a column offset by 1e3) against a direct-difference LAPACK reference, each bar a written
    formula with the measured ratio beside it;
B5. gpmpc_nlml at the corners and edge midpoints of the fit's bounds (optimize.bounds_and_init), fixed_bounds on and
    off: value and gradient where cond <= 1e12, LinAlgError exactly where the reference's jittered Cholesky fails;
B6. exact invariance under power-of-two rescaling of X, Z and ell, through every predict, derivative, EM, LOO and NLML
    path;
B7. appends and removals keep the K build's centre on the mean of the current X: a handle reached by appends and
    removals computes what a fresh set_data handle on the same X computes, bit for bit.

The bounds are written formulas (tests/_kernel_range.py), checked on the CPU in test_kernel_range_cpu.py."""
import math

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests import _kernel_range as kr
from tests._engines import ks_chunk

pytestmark = pytest.mark.gpu

SFS = (2.0 ** -20, 1.0, 2.0 ** 6 * 3)


def _engine(X, Y, hyper, capacity=None, factorize=True):
    import gp_mpc_b200
    eng = gp_mpc_b200.Engine(X.shape[0], X.shape[1], Y.shape[1], device=0, capacity=capacity)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)
    if factorize:
        eng.factorize()
    return eng


def _hyper(ell, sf, sn, Ny=1):
    return np.tile(np.concatenate([ell, [sf, sn]]), (Ny, 1))


def entry_ref(tex, dt):
    """Reference value and allowed error of device entries 2^t~ whose exact exponent is tex (long double) and whose
    computed t~ is within dt of it: 2^-1020 exactly below the clamp, k* (1 +- rel_bound) above it, either in between."""
    tex = np.asarray(tex); dt = np.asarray(dt, dtype=np.float64)
    kex = kr.k_exact(tex)
    below = tex < kr.T_MIN - dt
    above = tex > kr.T_MIN + dt
    ref = np.where(below, kr.K_MIN, kex).astype(np.float64)
    tol = np.where(below, 0.0, (kex * kr.rel_bound(dt)).astype(np.float64))
    band = ~below & ~above
    tol = np.where(band, np.abs(kr.K_MIN - kex).astype(np.float64) + (kex * kr.rel_bound(dt)).astype(np.float64), tol)
    return ref, tol, below


def _check_K(K, X, ell, sf, mu):
    """Off-diagonal entries of a device K against entry_ref: (worst error / allowed, number of clamped entries)."""
    N = X.shape[0]
    tex = kr.t_exact(X, X, ell, sf)
    _, dt, _, _ = kr.kbuild_t(X, X, mu, ell, sf * sf)
    ref, tol, below = entry_ref(tex, dt)
    off = ~np.eye(N, dtype=bool)
    assert np.all(K[below & off] == kr.K_MIN)            # the clamp's documented result, bit for bit
    err = np.abs(K - ref)[off]
    allowed = tol[off]
    ok = err <= allowed
    assert ok.all(), (np.argwhere(~ok)[:5], err[~ok][:5], allowed[~ok][:5])
    return float(np.max(np.where(allowed > 0, err / np.where(allowed > 0, allowed, 1), 0))), int(np.sum(below & off))


def _designs_k():
    """(name, X, ell): the 1-D grid's spacing makes t run from log2 sf2 down past -1020; the Nx designs mix length scales
    per dimension so pairs land everywhere between.  Two exact duplicates sit in different 128-tiles (rows 3 and 200),
    where the tile takes no upper clamp."""
    rng = np.random.default_rng(21)
    out = []
    x = np.cumsum(rng.uniform(0.0, 0.4, 300))[:, None]                   # span ~60 ell: t down to ~-2600
    x[200] = x[3]
    out.append(('grid1d', x, np.array([1.0])))
    for Nx in (8, 17, 32):
        X = rng.standard_normal((300, Nx)) * np.where(np.arange(300) % 2 == 0, 0.5, 6.0)[:, None]
        X[200] = X[3]
        ell = np.exp(rng.uniform(np.log(0.3), np.log(3.0), Nx))
        out.append(('nx%d' % Nx, X, ell))
    return out


@pytest.mark.parametrize('sf', SFS)
@pytest.mark.parametrize('design', range(4))
def test_K_entries_across_the_exponent_range(design, sf):
    """Every off-diagonal entry within entry_ref's allowance, the clamped ones bit for bit; each design has entries below
    the clamp."""
    name, X, ell = _designs_k()[design]
    sn = 1e-3 * sf
    Y = np.zeros((X.shape[0], 1)); Y[0] = 1.0
    eng = _engine(X, Y, _hyper(ell, sf, sn), factorize=False)
    K = eng.build_K(0)
    eng.close()
    assert np.array_equal(K, K.T)                                          # bitwise symmetric, diagonal tiles too
    mu = X.mean(0)
    _, nclamp = _check_K(K, X, ell, sf, mu)
    assert nclamp > 0, name
    sf2, sn2 = sf * sf, sn * sn
    _, dt, _, _ = kr.kbuild_t(X, X, mu, ell, sf2)
    # diagonal: t_ii is log2 sf2 up to the expansion's rounding, clamped from above at the device's log2(sf2), whose exp2
    # is sf2 to EXP2_ULP ulp plus ln 2 ulp(log2 sf2) (up to ~11 eps at sf = 2^6 3): so K_ii may exceed sf2 + sn2 by that
    d = np.diag(K)
    dd = np.diag(dt)
    lg = math.log(2) * kr.ulp(math.log2(sf2))                            # the device log2's rounding, carried by exp2
    lo = (sf2 + sn2) - sf2 * (kr.rel_bound(dd) + lg) - 2 * kr.EPS * (sf2 + sn2)
    hi = (sf2 + sn2) + sf2 * (kr.EXP2_ULP * kr.EPS + lg) + 2 * kr.EPS * (sf2 + sn2)
    assert np.all(d >= lo) and np.all(d <= hi), (np.min(d - lo), np.max(d - hi))
    # duplicates in different tiles (no upper clamp there): k <= sf2 (1 + bound), same value as the diagonal's kernel part
    k32 = K[200, 3]
    assert k32 <= sf2 * (1 + kr.rel_bound(dt[200, 3])), (k32, sf2)
    assert abs(k32 - sf2) <= sf2 * kr.rel_bound(dt[200, 3])


def _sparse_grid(N, rng):
    """A 1-D grid with gaps of 6.6 to 8 ell: every off-diagonal entry is below 2^-30 sf2 (t <= log2 sf2 - 31)."""
    return np.cumsum(rng.uniform(6.6, 8.0, N))[:, None]


@pytest.mark.parametrize('sf', SFS)
def test_lower_build_through_L(sf):
    """kbuild_dmma_kernel<false> in both bodies: N = 384 has the diagonal tiles (checked body) and the off-diagonal
    tiles (1,0), (2,0), (2,1) that touch neither the diagonal nor the identity tail (unchecked body).  With every
    off-diagonal K_ij <= 2^-30 sf2 on an ordered grid, the terms L_ik L_jk (k < j < i) are below K_ij by 2^-120 or
    more, so (L L^T)_ij = L_ij L_jj = K_ij to rounding, and L_jj^2 = sf2 + sn2.  Subnormal L_ij (K_ij near 2^-1020 over
    L_jj > 1) carry an absolute rounding of 2^-1075."""
    rng = np.random.default_rng(31)
    X = _sparse_grid(384, rng)
    ell = np.array([1.0])
    sn = 0.1 * sf
    Y = rng.standard_normal((384, 1))
    eng = _engine(X, Y, _hyper(ell, sf, sn))
    Lc = eng.get(L.GET_CHOL, 0)
    eng.close()
    sf2, sn2 = sf * sf, sn * sn
    Ljj = np.diag(Lc)
    tex = kr.t_exact(X, X, ell, sf)
    _, dt, _, _ = kr.kbuild_t(X, X, X.mean(0), ell, sf2)
    lg = math.log(2) * kr.ulp(math.log2(sf2))
    # the grid spans ~2800 ell: |u|^2 ~ 3e6 from the centre, so K_jj itself carries ~1e-8 (the bound's diagonal)
    assert np.all(np.abs(Ljj * Ljj - (sf2 + sn2)) <= sf2 * (kr.rel_bound(np.diag(dt)) + lg) + 8 * kr.EPS * (sf2 + sn2))
    ref, tol, below = entry_ref(tex, dt)
    i, j = np.tril_indices(384, -1)
    assert np.all(tex[i, j] <= math.log2(sf2) - 30)
    assert np.any(below[i, j]) and np.any(tex[i, j] > kr.T_MIN + 100)
    # L L^T against the reference K, entry by entry (long double: no underflow in the check).  Above the clamp the
    # terms L_ik L_jk (k < j) are below K_ij by 2^-120 or more, so (L L^T)_ij is L_ij L_jj; where K_ij is clamped to
    # 2^-1020 they are ~2^-35 of it, and the Cholesky's backward error covers them.
    Ld = Lc.astype(kr.LD)
    LLt = (Ld @ Ld.T)[i, j]
    absL = np.abs(Ld)
    scale = (absL @ absL.T)[i, j].astype(np.float64)
    err = np.abs(LLt - ref[i, j]).astype(np.float64)
    allowed = tol[i, j] + 8 * kr.EPS * scale + 2.0 ** -1074 * 2 * (Ljj[j] + Ljj[i] + 1)
    assert np.all(err <= allowed), (np.argwhere(err > allowed)[:5], (err / allowed).max())
    assert np.all(np.triu(Lc, 1) == 0.0)


# ------------------------------------------------------------------ B3: ks values through predict
# (CH, Nx, outputs, N): every NXP each chunk size pairs with (launch_ks_nx: the next of 4, 6, 8, 10, 12, 16, 24, 32).
KS_RANGE_CASES = ([(1024, nx, 2, 8155) for nx in (3, 5, 8, 10, 12)] + [(512, nx, 1, 8155) for nx in (4, 5, 7, 9, 11)]
                  + [(512, nx, 2, 8155) for nx in (13, 20, 32)]
                  + [(128, nx, 2, 600) for nx in (2, 6, 8, 10, 12, 15, 20, 32)])
SPACING = 40.0          # lattice spacing in units of each dimension's ell: off-diagonal t <= -0.72 * 1600 = -1154, K = (sf2 + sn2) I + 2^-1020


def _lattice(N, Nx, rng):
    """N training points on a lattice of spacing 40 ell in dims 0 .. m-1 (m = min(3, Nx - 1)), small offsets in the
    other dims but the last, which is 0: the test points sweep along the last dim, away from every training point."""
    m = min(3, Nx - 1)
    side = int(math.ceil(N ** (1.0 / m)))
    idx = np.array(np.unravel_index(np.arange(N), (side,) * m)).T
    X = np.zeros((N, Nx))
    X[:, :m] = (idx - side // 2) * SPACING
    if Nx - 1 > m:
        X[:, m:Nx - 1] = rng.uniform(-0.5, 0.5, (N, Nx - 1 - m))
    return X


@pytest.mark.parametrize('ch,Nx,Ny,N', KS_RANGE_CASES)
def test_ks_values_one_by_one(ch, Nx, Ny, N):
    """Output a has target one-hot at training point j_a; test points z = x_j + s ell_last e_last (+ small offsets) with s
    from 0 to 46, so t runs from log2 sf2 to below -1020.  mean = sum_i alpha_i ks_i(z), dominated by i = j, is checked
    against the same sum over reference entries (entry_ref) within sum_i |alpha_i| tol_i; J likewise per component,
    where the scaled difference adds an absolute u_r (|xs| + |zs|) per dimension and, at sf = 3 2^6 (alpha ~ 3e-5),
    the terms alpha_i 2^-1020 are subnormal and carry an absolute rounding of 2^-1075 per fma; var = sf2 - |L^-1 ks|^2 within its
    cancellation-aware bound."""
    assert ks_chunk(-(-N // 128) * 128, Ny, Nx) == ch
    rng = np.random.default_rng(1000 + 10 * Nx + Ny + ch)
    ell = np.exp(rng.uniform(np.log(0.05), np.log(20.0), Nx))          # a different length scale per dimension
    X = _lattice(N, Nx, rng) * ell
    sf = SFS[Nx % 3]
    sn = 1e-2 * sf
    js = rng.choice(N, Ny, replace=False)
    Y = np.zeros((N, Ny))
    for a, j in enumerate(js):
        Y[j, a] = 1.0
    eng = _engine(X, Y, _hyper(ell, sf, sn, Ny))
    s = np.linspace(0.0, 46.0, 48)
    sf2 = sf * sf
    for a, j in enumerate(js):
        Z = np.repeat(X[j][None, :], s.size, 0)
        Z[:, -1] += s * ell[-1]
        if Nx > 1:
            Z[:, 0] += rng.uniform(-0.3, 0.3, s.size) * ell[0]
        mean, var, _, jac = eng.predict(Z, np.zeros((Nx, Nx)), L.METHOD_TA)
        alpha = eng.get(L.GET_ALPHA, a)
        linv = eng.get(L.GET_LINV, a)
        tex = kr.t_exact(X, Z, ell, sf)                                   # (N, H)
        _, dt = kr.ks_t(X, Z, ell, sf2)
        ref, tol, below = entry_ref(tex, dt)
        assert below[j].any() and (tex[j] > math.log2(sf2) - 20).any()
        w = alpha[:, None] * ref
        m_ref = w.sum(0)
        m_tol = np.abs(alpha) @ tol + 8 * kr.EPS * np.abs(w).sum(0)
        assert np.all(np.abs(mean[:, a] - m_ref) <= m_tol), (np.abs(mean[:, a] - m_ref) / m_tol).max()
        # single term: the others are below alpha_j ks_j by 2^-100 or more wherever ks_j is above the clamp
        top = tex[j] > -900
        assert np.all(np.abs(m_ref[top] - w[j, top]) <= 1e-12 * np.abs(w[j, top]))
        D = (X[:, None, :] - Z[None, :, :]) / ell                          # exact in these designs' ranges to u_r
        xs, zs = np.abs(X / ell), np.abs(Z / ell)
        dif = 2 * kr.EPS * (xs[:, None, :] + zs[None, :, :] + np.abs(D))      # absolute error of xs - zs
        J_ref = np.einsum('nh,nhd->hd', w, D / ell)
        J_tol = (np.einsum('nh,nhd->hd', np.abs(alpha)[:, None] * (tol + ref * 8 * kr.EPS), np.abs(D) / ell)
                 + np.einsum('nh,nhd->hd', np.abs(w), dif / ell)
                 + 4 * N * 2.0 ** -1074 * (1 + np.max(np.abs(D), axis=0) / ell))    # subnormal w: 2^-1075 per fma
        bad = np.argwhere(np.abs(jac[:, a, :] - J_ref) > J_tol)
        assert bad.size == 0, (bad[:4], jac[:, a, :][tuple(bad[0])], J_ref[tuple(bad[0])], J_tol[tuple(bad[0])])
        v = linv @ ref
        v_tol = linv.__abs__() @ tol
        var_ref = sf2 - np.einsum('nh,nh->h', v, v)
        var_tol = 2 * np.einsum('nh,nh->h', np.abs(v), v_tol) + 8 * kr.EPS * (sf2 + np.einsum('nh,nh->h', v, v)) \
            + 2 * kr.EPS * sf2
        assert np.all(np.abs(var[:, a] - var_ref) <= var_tol), (np.abs(var[:, a] - var_ref) / var_tol).max()
    eng.close()


# ------------------------------------------------------------------ B6: power-of-two rescaling
@pytest.mark.parametrize('s', (2.0 ** 7, 2.0 ** -7))
def test_power_of_two_rescaling_is_exact(s):
    """X, Z and ell scaled by s = 2^+-7 and Sigma by s^2: host mu, 1/ell, the centred u, the direct differences and
    every product with 1/ell scale exactly, so K, L, L^-1, alpha, mean, var, the TA, ME and EM covariances, the LOO
    predictions and the NLML are the same bits; every derivative w.r.t. z scales by exactly s^-k for its order k (J,
    dvar_dz and dcov_dz by 1/s, the mean Hessian and the second derivatives of var and cov by 1/s^2, d3mean_dz3 by
    1/s^3), the EM derivatives w.r.t. Sigma by 1/s^2, and the NLML's ell-gradient by 1/s.  An absolute constant in any
    of these kernels would break the equality."""
    p = orc.synthetic_problem(700, 6, 2, config_id=61, H=40)
    X, Y, hyper, Z, Sigma = p['X'], p['Y'], p['hyper'].copy(), p['Z'], p['Sigma']
    hs = hyper.copy(); hs[:, :6] *= s
    e1 = _engine(X, Y, hyper)
    e2 = _engine(X * s, Y, hs)
    for what in (L.GET_CHOL, L.GET_LINV, L.GET_ALPHA):
        for a in (0, 1):
            assert np.array_equal(e1.get(what, a), e2.get(what, a)), (what, a)
    assert np.array_equal(e1.build_K(1), e2.build_K(1))
    m1, v1, c1, J1 = e1.predict(Z, Sigma, L.METHOD_TA)
    m2, v2, c2, J2 = e2.predict(Z * s, Sigma * s * s, L.METHOD_TA)
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2) and np.array_equal(c1, c2)
    assert np.array_equal(J1, J2 * s)
    for x1, x2 in zip(e1.loo(), e2.loo()):
        assert np.array_equal(x1, x2)
    m1, v1, c1, _ = e1.predict(Z, Sigma, L.METHOD_ME)
    m2, v2, c2, _ = e2.predict(Z * s, Sigma * s * s, L.METHOD_ME)
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2) and np.array_equal(c1, c2)
    m1, v1, c1, _ = e1.predict(Z, Sigma, L.METHOD_EM, want_jac=False)
    m2, v2, c2, _ = e2.predict(Z * s, Sigma * s * s, L.METHOD_EM, want_jac=False)
    assert np.array_equal(m1, m2) and np.array_equal(v1, v2) and np.array_equal(c1, c2)
    # derivatives w.r.t. z scale by 1/s per order, w.r.t. Sigma by 1/s^2
    scaling = dict(mean=0, var=0, cov=0, jac=1, dvar_dz=1, dcov_dz=1, hess=2, d2var_dz2=2, d2cov_dz2=2, d3mean_dz3=3,
                   dmean_dz=1, dmean_dSigma=2, dcov_dSigma=2)
    for method in (L.METHOD_TA, L.METHOD_ME):
        r1 = e1.predict_hess(Z, Sigma, method)
        r2 = e2.predict_hess(Z * s, Sigma * s * s, method)
        for k, v in r1.items():
            assert np.array_equal(v, r2[k] * s ** scaling[k]), (method, k)
    r1 = e1.predict_em_grad(Z, Sigma)
    r2 = e2.predict_em_grad(Z * s, Sigma * s * s)
    for k, v in r1.items():
        assert np.array_equal(v, r2[k] * s ** scaling[k]), ('EM', k)
    n1, g1 = e1.nlml(0, hyper[0])
    n2, g2 = e2.nlml(0, hs[0])
    assert n1 == n2 and np.array_equal(g1[6:], g2[6:]) and np.array_equal(g1[:6], g2[:6] * s)
    e1.close(); e2.close()


# ------------------------------------------------------------------ B7: the centre follows appends and removals
@pytest.mark.parametrize('greedy', (False, True))
def test_centre_follows_appends_and_removals(greedy):
    """A reserved handle at N0 = 256 around 0, factorised; 512 points shifted by c = 1e3 in column 0 appended (one by
    one, or by greedy selection from a pool of 600); the original 256 removed; set_hyper and factorize.  The handle
    must compute what a fresh set_data handle on the same X and Y (same order, same capacity) computes, bit for bit:
    K, L, alpha, log det, nlml and loo_nlpp; and every entry of its K must meet the direct-difference reference at the
    bound for a centre at the current mean.  With the centre left at the old mean, |u|^2 reaches ~6e5 and the bound on
    t grows ten-thousandfold."""
    rng = np.random.default_rng(77)
    Nx, N0, n_new = 4, 256, 512
    X0 = rng.standard_normal((N0, Nx))
    pool = rng.standard_normal((600 if greedy else n_new, Nx)) * 1.5
    pool[:, 0] += 1e3
    f = lambda x: np.sin(x[:, 1:2]) + 0.1 * x[:, 0:1] - 100.0 * (x[:, 0:1] > 500)
    Y0, Yp = f(X0), f(pool)
    hyper = _hyper(np.array([1.5, 1.0, 2.0, 1.2]), 1.0, 1e-2)
    cap = N0 + n_new
    eng = _engine(X0, Y0, hyper, capacity=cap)
    if greedy:
        picked, _, ok = eng.append_greedy(pool, Yp, n_new)
        assert ok and picked.size == n_new
        Xn, Yn = pool[picked], Yp[picked]
    else:
        for x, y in zip(pool, Yp):
            assert eng.append(x, y)
        Xn, Yn = pool, Yp
    eng.remove(np.arange(N0))
    assert eng.N == n_new
    eng.set_hyper(hyper)
    eng.factorize()
    fresh = _engine(Xn, Yn, hyper, capacity=cap)
    for what in (L.GET_CHOL, L.GET_ALPHA, L.GET_LOGDET):
        assert np.array_equal(eng.get(what, 0), fresh.get(what, 0)), what
    assert np.array_equal(eng.build_K(0), fresh.build_K(0))
    n1, g1 = eng.nlml(0, hyper[0]); n2, g2 = fresh.nlml(0, hyper[0])
    assert n1 == n2 and np.array_equal(g1, g2)
    l1, h1 = eng.loo_nlpp(0, hyper[0]); l2, h2 = fresh.loo_nlpp(0, hyper[0])
    assert l1 == l2 and np.array_equal(h1, h2)
    # every entry of K against the long-double direct-difference reference, within the bound for the centre at the
    # mean of the current X (a centre left at the old mean breaks it by orders of magnitude: |u|^2 ~ 6e5 instead of ~60)
    ell = hyper[0, :Nx]
    _check_K(eng.build_K(0), Xn, ell, 1.0, Xn.mean(0))
    eng.close(); fresh.close()


# ------------------------------------------------------------------ B4: regimes end to end
# Reference: K by direct differences (oracle covSEard; the oracle's assemble_K uses the un-centred expansion, whose own
# error at a column offset of 1e3 would swamp the comparison) plus sn2 I, LAPACK Cholesky with the single 1e-8 jitter
# retry.  Bars, all written formulas: with kappa = cond_2(K), U = 1 + max |u|^2 from the centre, rho the K build's
# largest entry bound (kbuild_bound at U) and c = kappa (rho + N eps) the norm-wise relative perturbation of K^-1 that
# rho and both factorisations' backward errors allow:
#   alpha, L: relative 2-norm / Frobenius error <= 4 c (sqrt(N) for L);  log det: <= 2 N c;
#   mean, J: <= 4 rho_ks sum |terms| + 4 c |alpha|_2 |ks-term|_2 + 2^-1019 |alpha|_1 (|D|)  (rho_ks the ks kernel's
#         largest entry bound; the last term is the clamp where the reference underflows);
#   var: <= 4 rho_ks |ks|_2 |v|_2 + 4 c |v|_2^2 lambda_max + 8 eps sf2 + 2^-1019 |v|_1 (v = K^-1 ks);
#   NLML value: <= 4 c (|y|_2 |alpha|_2 + N);  gradient component d: <= 4 c sum_ij (|K^-1| + |alpha alpha^T|) |dK_d|.
# The derivative, EM and LOO paths are held to 64 c (1 + r2)^(3/2) of their largest reference entry, r2 the largest
# |(x - z)/ell|^2 that carries weight.
# Measured ratios to these bars on an H100 SXM (80 GB HBM3, 700 W), largest over both outputs and TA / ME:
#   short_ell: mean, J 1.1e-5, alpha 9e-7, L 3.7e-7, nlml 1.7e-7, nlml_grad 9.2e-6, derivatives / EM / LOO <= 8.8e-9
#   long_ell:  alpha 2.1e-4, logdet 2.4e-6, nlml 3.9e-6, nlml_grad 5.2e-5, the rest <= 1.5e-10
#   ard:       J 2.8e-2, mean 3.4e-3, alpha 2.3e-5, nlml_grad 4.4e-6, derivatives / EM / LOO <= 1.1e-8
#   sf 3 2^-10: alpha 5.5e-5, nlml_grad 4.4e-5, em_cov 6e-6, L 2.1e-6, the rest <= 1.2e-6
#   sf 3 2^10: alpha 5.8e-5, em_cov 4.2e-5, nlml_grad 1.9e-5, em_dcov_dz 1.1e-5, logdet 8e-6, the rest <= 2e-6
#   offset:    alpha 5.8e-5, nlml_grad 1.2e-5, the rest <= 4.4e-7
# The bars carry cond(K), which is 1e4 to 1e10 here, so they are loose where K is ill-conditioned; the K entries
# themselves are held to their own bounds, entry by entry, in test_K_entries_across_the_exponent_range.
def _regimes():
    rng = np.random.default_rng(404)
    N, Nx = 400, 4
    X = rng.standard_normal((N, Nx))
    out = []
    out.append(('short_ell', X, np.array([[0.03, 0.05, 0.04, 0.03, 1.0, 1e-2], [0.05, 0.03, 0.03, 0.05, 1.0, 1e-2]]), True))
    out.append(('long_ell', X, np.array([[30.0, 40.0, 30.0, 50.0, 1.0, 1e-5], [60.0, 30.0, 40.0, 30.0, 1.0, 1e-5]]), False))
    out.append(('ard', X, np.array([[1e-2, 1.0, 1e2, 1e4, 1.0, 1e-2], [1e4, 0.5, 3.0, 1e-1, 1.0, 1e-2]]), True))
    for sf in (2.0 ** -10 * 3, 2.0 ** 10 * 3):
        out.append(('sf%g' % sf, X, np.array([[1.5, 2.0, 1.0, 2.5, sf, 1e-5 * sf], [2.0, 1.5, 2.5, 1.0, sf, 0.5 * sf]]),
                    True))
    Xo = X.copy(); Xo[:, 0] += 1e3
    out.append(('offset', Xo, np.array([[1.5, 2.0, 1.0, 2.5, 1.0, 1e-2], [2.0, 1.5, 2.5, 1.0, 1.0, 1e-2]]), False))
    return out


def _ref_model(X, Y, hyper):
    """Per output: dict(K (with the jitter used), L, Linv, alpha, jit) from direct differences and LAPACK."""
    from scipy.linalg import solve_triangular
    Nx = X.shape[1]
    out = []
    for a in range(hyper.shape[0]):
        K = orc.covSEard(X, X, hyper[a, :Nx], hyper[a, Nx] ** 2) + hyper[a, Nx + 1] ** 2 * np.eye(X.shape[0])
        Lr, jit = orc.chol_with_jitter(K)
        if jit:
            K = K + 1e-8 * np.eye(X.shape[0])
        Li = solve_triangular(Lr, np.eye(X.shape[0]), lower=True)
        out.append(dict(K=K, L=Lr, Li=Li, alpha=Li.T @ (Li @ Y[:, a]), jit=jit))
    return out


def _c_bar(X, hyper_a, K):
    Nx = X.shape[1]
    lam = np.linalg.eigvalsh(K)
    Ui = (X - X.mean(0)) * kr.SQRT_LOG2E / hyper_a[:Nx]
    U = 1 + np.max(np.sum(Ui * Ui, 1))
    rho = kr.rel_bound((Nx + 6) * kr.EPS * (3 * U + abs(math.log2(hyper_a[Nx] ** 2))) + 4 * kr.EPS)
    return lam[-1] / lam[0] * (rho + X.shape[0] * kr.EPS), lam, rho


@pytest.mark.parametrize('regime', range(6))
def test_regimes_end_to_end(regime):
    """factorize (L, alpha, log det and the jitter decision), predict TA / ME (mean, var, J, cov) and nlml with its
    gradient against the direct-difference reference, each within its written bar (see above); for the short-ell, ARD
    and sf regimes also predict_hess, predict_em_grad, loo and loo_nlpp."""
    from oracle import em_grad_oracle as emo
    from oracle import hess_oracle as hso
    from oracle import loo_oracle as loo
    name, X, hyper, extra = _regimes()[regime]
    N, Nx = X.shape
    rng = np.random.default_rng(405 + regime)
    Y = np.stack([np.sin(X[:, 1] / hyper[0, 1]) + 0.1 * rng.standard_normal(N),
                  np.cos(X[:, 2] / hyper[1, 2]) + 0.1 * rng.standard_normal(N)], 1) * hyper[:, Nx]
    Z = X[:20] + rng.standard_normal((20, Nx)) * hyper[0, :Nx] * (4.0 if name == 'short_ell' else 0.3)
    Sigma = np.diag(hyper[0, :Nx] ** 2) * 1e-3
    eng = _engine(X, Y, hyper, factorize=False)
    info = eng.factorize()
    ref = _ref_model(X, Y, hyper)
    ratios = {}

    def chk(key, err, bar):
        err, bar = np.broadcast_arrays(np.asarray(err, dtype=np.float64), np.asarray(bar, dtype=np.float64))
        r = float(np.max(np.where(bar > 0, err / np.where(bar > 0, bar, 1.0), np.where(err > 0, np.inf, 0.0))))
        ratios[key] = max(ratios.get(key, 0.0), r)
        assert r <= 1.0, (name, key, r)

    res = {m: eng.predict(Z, Sigma, m) for m in (L.METHOD_TA, L.METHOD_ME)}
    for a in range(2):
        R = ref[a]
        assert bool(info[a]) == bool(R['jit']), (name, a, info[a], R['jit'])       # the same jitter decision
        c, lam, _ = _c_bar(X, hyper[a], R['K'])
        al = eng.get(L.GET_ALPHA, a)
        chk('alpha', np.linalg.norm(al - R['alpha']), 4 * c * np.linalg.norm(R['alpha']))
        chk('L', np.linalg.norm(eng.get(L.GET_CHOL, a) - R['L']), 4 * c * math.sqrt(N) * np.linalg.norm(R['L'], 2))
        ld = 2 * np.sum(np.log(np.diag(R['L'])))
        chk('logdet', abs(eng.get(L.GET_LOGDET, a)[0] - ld), 2 * N * c + 8 * kr.EPS * abs(ld))
        ell, sf2 = hyper[a, :Nx], hyper[a, Nx] ** 2
        _, dts = kr.ks_t(X, Z, ell, sf2)
        rks = float(np.max(kr.rel_bound(dts)))
        ks = orc.covSEard(X, Z, ell, sf2)                                      # (N, H)
        w = R['alpha'][:, None] * ks
        D = (X[:, None, :] - Z[None, :, :]) / ell ** 2                         # (N, H, Nx)
        v = R['Li'].T @ (R['Li'] @ ks)
        var_ref = sf2 - np.sum(ks * v, 0)
        J_ref = np.einsum('nh,nhd->hd', w, D)
        na = np.linalg.norm(R['alpha'])
        flo = 2 * kr.K_MIN * np.abs(R['alpha']).sum()                     # where the reference underflows below the clamp
        m_bar = 4 * rks * np.abs(w).sum(0) + 4 * c * na * np.linalg.norm(ks, axis=0) + flo
        J_bar = 4 * rks * np.einsum('nh,nhd->hd', np.abs(w), np.abs(D)) \
            + 4 * c * na * np.linalg.norm(ks[:, :, None] * D, axis=0) + flo * np.max(np.abs(D), axis=0)
        v_bar = 4 * rks * np.linalg.norm(ks, axis=0) * np.linalg.norm(v, axis=0) \
            + 4 * c * np.sum(v * v, 0) * lam[-1] + 8 * kr.EPS * sf2 + 2 * kr.K_MIN * np.abs(v).sum(0)
        for m in (L.METHOD_TA, L.METHOD_ME):
            mean, var, cov, jac = res[m]
            chk('mean', np.abs(mean[:, a] - w.sum(0)), m_bar)
            chk('var', np.abs(var[:, a] - var_ref), v_bar)
            chk('J', np.abs(jac[:, a] - J_ref), J_bar)
            cdiag = var_ref + (np.einsum('hd,de,he->h', J_ref, Sigma, J_ref) if m == L.METHOD_TA else 0)
            c_bar = v_bar + (2 * np.einsum('hd,de,he->h', J_bar, np.abs(Sigma), np.abs(J_ref) + J_bar)
                             if m == L.METHOD_TA else 0)
            chk('cov', np.abs(cov[:, a, a] - cdiag), c_bar + 8 * kr.EPS * np.abs(cdiag))
        # NLML value and gradient at the model's own hyper-parameters
        Ki = R['Li'].T @ R['Li']
        nll_ref = 0.5 * Y[:, a] @ R['alpha'] + 0.5 * ld
        nll, g = eng.nlml(a, hyper[a])
        eng.factorize()                                                        # nlml uses the factor's slabs as scratch
        chk('nlml', abs(nll - nll_ref), 4 * c * (np.linalg.norm(Y[:, a]) * na + N) + 8 * kr.EPS * abs(nll_ref))
        Kf = orc.covSEard(X, X, ell, sf2)
        Wm = Ki - np.outer(R['alpha'], R['alpha'])
        Wa = np.abs(Ki) + np.abs(np.outer(R['alpha'], R['alpha']))
        dK = [Kf * (X[:, d][:, None] - X[:, d][None, :]) ** 2 / ell[d] ** 3 for d in range(Nx)]
        dK += [2 * Kf / hyper[a, Nx], 2 * hyper[a, Nx + 1] * np.eye(N)]
        g_ref = np.array([0.5 * np.sum(Wm * dk) for dk in dK])
        g_bar = np.array([4 * c * 0.5 * np.sum(Wa * np.abs(dk)) for dk in dK])
        chk('nlml_grad', np.abs(g - g_ref), g_bar + 8 * kr.EPS * np.abs(g_ref))
    if extra:
        alpha = np.stack([R['alpha'] for R in ref]); chol = np.stack([R['L'] for R in ref])
        c = max(_c_bar(X, hyper[a], ref[a]['K'])[0] for a in range(2))
        r2 = max(float(np.max(np.sum(((X[:, None, :] - Z[None, :, :]) / hyper[a, :Nx]) ** 2, -1)
                              * (orc.covSEard(X, Z, hyper[a, :Nx], 1.0) > 1e-16))) for a in range(2))
        gbar = 64 * c * (1 + r2) ** 1.5

        def chk_rel(key, got, want):
            chk(key, np.max(np.abs(got - want)), gbar * max(np.max(np.abs(want)), 1e-300))

        hr = hso.predict_hess(X, hyper, alpha, chol, Z, Sigma, method='TA')
        he = eng.predict_hess(Z, Sigma, L.METHOD_TA)
        for k_ref, k_eng in (('dvar', 'dvar_dz'), ('hess', 'hess'), ('d2var', 'd2var_dz2'), ('d3mean', 'd3mean_dz3'),
                             ('dcov', 'dcov_dz')):
            chk_rel(k_eng, he[k_eng], hr[k_ref])
        er = emo.em_grad_closed(X, hyper, alpha, chol, Z[:6], Sigma)
        ee = eng.predict_em_grad(Z[:6], Sigma)
        for k in ('mean', 'cov', 'dmean_dz', 'dmean_dSigma', 'dcov_dz', 'dcov_dSigma'):
            chk_rel('em_' + k, ee[k], er[k])
        lm, lv, lp = eng.loo()
        for a in range(2):
            Li = ref[a]['Li']; cc = np.sum(Li * Li, 0); r = ref[a]['alpha'] / cc
            chk_rel('loo_mean', lm[a], Y[:, a] - r)
            chk_rel('loo_var', lv[a], 1.0 / cc)
            f, gl = eng.loo_nlpp(a, hyper[a])
            nl = np.sum(0.5 * np.log(2 * np.pi) - 0.5 * np.log(cc) + 0.5 * ref[a]['alpha'] * r)
            chk('loo_nlpp', abs(f - nl), gbar * (1 + abs(nl)))
            g_or = loo.grad_trace(X, Y[:, a], hyper[a])
            chk_rel('loo_nlpp_grad', gl, g_or)
    eng.close()
    print('\n[B4 ratio to bar] %s: %s' % (name, ' '.join('%s=%.2g' % kv for kv in sorted(ratios.items()))))


# ------------------------------------------------------------------ B5: nlml on the fit's box
def _pivots(K):
    """Schur pivots of an unpivoted Cholesky of K up to and including the first non-positive one."""
    A = K.copy()
    out = []
    for k in range(A.shape[0]):
        p = A[k, k]
        out.append(p)
        if p <= 0:
            break
        l = A[k + 1:, k] / math.sqrt(p)
        A[k + 1:, k + 1:] -= np.outer(l, l)
    return np.array(out)


@pytest.mark.parametrize('fixed', (False, True))
def test_nlml_on_the_corners_and_edge_midpoints_of_the_fit_box(fixed):
    """gpmpc_nlml at every corner and edge midpoint of optimize.bounds_and_init's box (the ell lower bound is the
    replicated -1 unless fixed_bounds; the kernel sees ell^2), on standardised data.  Where the direct-difference K
    with the jitter its Cholesky needed has cond <= 1e12: the value within 4 c (|y| |alpha| + N) and each gradient
    component within 4 c sum (|K^-1| + |alpha alpha^T|) |dK_d| (c as in B4).  Elsewhere: the engine raises
    LinAlgError exactly when the reference's Cholesky fails after the 1e-8 jitter.  Points where a Schur pivot of the
    reference lies within 1e-6 (relative to its diagonal) of zero are skipped: there the two factorisations' rounding
    decides the outcome, not the kernel."""
    import itertools
    import gp_mpc_b200
    from gp_mpc_b200 import optimize as opt
    rng = np.random.default_rng(506)
    N, Nx = 160, 2
    X = rng.standard_normal((N, Nx))
    X = (X - X.mean(0)) / X.std(0)
    y = np.sin(2 * X[:, 0]) + 0.3 * X[:, 1]
    y = (y - y.mean()) / y.std()
    bounds, _ = opt.bounds_and_init(X, y, fixed_bounds=fixed)
    lb, ub = bounds[:, 0], bounds[:, 1]
    m = Nx + 2
    pts = set()
    for corner in itertools.product((0, 1), repeat=m):
        pts.add(tuple(float(c) for c in corner))
        for d in range(m):
            e = list(corner); e[d] = 0.5
            pts.add(tuple(e))
    eng = gp_mpc_b200.Engine(N, Nx, 1, device=0)
    eng.set_data(X, y[:, None])
    eng.set_hyper(np.concatenate([np.ones(Nx), [1.0, 0.1]])[None, :])
    compared = raised = skipped = 0
    for p in sorted(pts):
        th = lb + np.array(p) * (ub - lb)
        ell, sf, sn = th[:Nx], th[Nx], th[Nx + 1]
        Kf = orc.covSEard(X, X, ell, sf * sf)
        K = Kf + sn * sn * np.eye(N)
        piv = _pivots(K)
        fails = piv[-1] <= 0
        if fails:
            Kj = K + 1e-8 * np.eye(N)
            piv = _pivots(Kj)
            fails = piv[-1] <= 0
            K = Kj
        diag = np.diag(K)[:piv.size]
        if np.any(np.abs(piv) <= 1e-6 * diag):
            skipped += 1
            continue
        if fails:
            with pytest.raises(np.linalg.LinAlgError):
                eng.nlml(0, th)
            raised += 1
            continue
        nll, g = eng.nlml(0, th)
        lam = np.linalg.eigvalsh(K)
        if lam[-1] / lam[0] > 1e12:
            continue
        Lr = np.linalg.cholesky(K)
        from scipy.linalg import cho_solve
        alpha = cho_solve((Lr, True), y)
        Ki = cho_solve((Lr, True), np.eye(N))
        c, _, _ = _c_bar(X, th, K)
        nll_ref = 0.5 * y @ alpha + np.sum(np.log(np.diag(Lr)))
        assert abs(nll - nll_ref) <= 4 * c * (np.linalg.norm(y) * np.linalg.norm(alpha) + N) + 8 * kr.EPS * abs(nll_ref)
        Wm = Ki - np.outer(alpha, alpha)
        Wa = np.abs(Ki) + np.abs(np.outer(alpha, alpha))
        dK = [Kf * (X[:, d][:, None] - X[:, d][None, :]) ** 2 / ell[d] ** 3 for d in range(Nx)]
        dK += [2 * Kf / sf, 2 * sn * np.eye(N)]
        for d, dk in enumerate(dK):
            gr = 0.5 * np.sum(Wm * dk)
            assert abs(g[d] - gr) <= 4 * c * 0.5 * np.sum(Wa * np.abs(dk)) + 8 * kr.EPS * abs(gr), (p, d, g[d], gr)
        compared += 1
    eng.close()
    print('\n[B5 fixed_bounds=%s] compared %d, raised %d, skipped %d of %d' % (fixed, compared, raised, skipped, len(pts)))
    assert compared > 0

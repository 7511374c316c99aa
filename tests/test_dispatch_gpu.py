"""The kernel instantiations the engine selects from the padded size Npad, Nx and the number of outputs on a handle, each
against a float64 reference:

A. the ks kernel's training-point chunk CH (ks_chunk, gpmpc.cu:807-811) with every register extent NXP it pairs with
   (launch_ks_nx, gpmpc.cu:957-972), checked on the engine's own alpha and L^-1 so the ks kernel and the predict product
   are tested alone;
B. the factorisation's recursion splits (potrf_inv_rec, gpmpc.cu:229-333) and the three GEMM feeds of gemm128
   (gpmpc.cu:204-219: 64x32 cp.async, 128x64 cp.async, 128x64 TMA tensor maps), against LAPACK on the engine's own K;
C. the NLML value and gradient (nlml_grad_kernel<8/16/32>, nxp_dispatch gpmpc.cu:188-196) and K^-1 (compute_kinv).

Sums that cancel (mean, Jacobian, NLML gradient) are normalised by the sum of the absolute values of their terms: alpha
alternates in sign and is conditioning-limited, so an error relative to the result would hide a kernel error behind
cancellation.  Every factorisation case also runs on a well-conditioned variant (sn = 0.3), where the bars are orders of
magnitude tighter than the conditioning-limited ones of the synthetic problem (sn = 1e-2).  The measured errors quoted
in the tests are from an H100 SXM (80 GB HBM3, 132 SMs) at its 700 W power limit."""
import numpy as np
import pytest
from scipy.linalg import cho_solve, solve_triangular

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle import hess_oracle as hso
from tests._engines import fit, gemm_feed, ks_chunk, npad, require, sms
from tests._util import relinf

pytestmark = pytest.mark.gpu

MAX_DEPTH, LOOKAHEAD_MIN_ROWS, LEAF_N = 12, 1024, 128        # gpmpc.cu:26-27, kernels.cuh:206
N_KS = 8155                                                    # Npad 8192, the last 1024-point chunk is partial


# ------------------------------------------------------------------ shape selection


def factor_products(n, depth=0):
    """The GEMMs of potrf_inv_rec (gpmpc.cu:241-331) on an n-row block: (step, mt, nt, lower, bt, n1, n2, h2)."""
    if n <= LEAF_N:
        return []
    nb = n // 128
    n1 = (nb // 2) * 128
    n2 = n - n1
    h2 = ((n2 // 128) // 2) * 128
    split = depth < MAX_DEPTH and h2 >= 128 and n >= LOOKAHEAD_MIN_ROWS
    sz = (n1, n2, h2)
    out = factor_products(n1, depth + 1)
    if split:
        out += [('panel', h2 // 128, n1 // 128, 0, True) + sz, ('update', h2 // 128, h2 // 128, 1, True) + sz,
                ('panel', (n2 - h2) // 128, n1 // 128, 0, True) + sz, ('update', (n2 - h2) // 128, h2 // 128, 0, True) + sz,
                ('update', (n2 - h2) // 128, (n2 - h2) // 128, 1, True) + sz]
    else:
        out += [('panel', n2 // 128, n1 // 128, 0, True) + sz, ('update', n2 // 128, n2 // 128, 1, True) + sz]
    out += [('w2', n2 // 128, n1 // 128, 0, False) + sz]
    out += factor_products(n2, depth + 1)
    out += [('li21', n2 // 128, n1 // 128, 0, False) + sz]
    return out


def factor_feeds(npad, batch, sms, small_tiles=None):
    """Per product of an Npad-row factorisation of `batch` outputs: (step, feed, tiles, lower, n1, n2, h2)."""
    out = []
    for step, mt, nt, lower, bt, n1, n2, h2 in factor_products(npad):
        feed, tiles = gemm_feed(mt, nt, lower, bt, batch, sms, small_tiles)
        out.append((step, feed, tiles, lower, n1, n2, h2))
    return out


# ------------------------------------------------------------------ A. ks kernel buckets (predict path)
# (CH, Nx, outputs, N): CH = 1024 needs Npad >= 8192, two outputs and Nx <= 12; CH = 512 the same Npad with one output or
# Nx > 12; CH = 128 is every Npad below 8192.  NXP (launch_ks_nx, gpmpc.cu:960-969) is the next of 4, 6, 8, 10, 12, 16, 24,
# 32 at or above Nx.  At Nx = 32 the kernel's final reduction has 8 x 33 values for its 256 threads.
KS_CASES = ([(1024, nx, 2, N_KS) for nx in (3, 5, 8, 10, 12)] + [(512, nx, 1, N_KS) for nx in (4, 6, 8, 12)]
            + [(512, nx, 2, N_KS) for nx in (13, 20, 32)] + [(128, 15, 2, 1000), (128, 32, 1, 1000)])


def _ks_problem(N, Nx, Ny):
    p = orc.synthetic_problem(N, Nx, Ny, config_id=100 + Nx + Ny, H=70)
    return p['X'], p['Y'], p['hyper'], p['Z'], p['Sigma']


def ks_reference(X, hyper_a, alpha, linv, Z):
    """mean = ks^T alpha, J = sum_i alpha_i ks_i (x_i - z) / ell^2 and var = sf2 - |L^-1 ks|^2 with ks by direct
    differences and np.exp, plus the sums of |terms| of mean and J."""
    Nx = X.shape[1]
    ell = hyper_a[:Nx]; sf2 = hyper_a[Nx] ** 2
    D = (X[:, None, :] - Z[None, :, :]) / ell                     # (N, H, Nx)
    ks = sf2 * np.exp(-0.5 * np.einsum('nhd,nhd->nh', D, D))
    w = alpha[:, None] * ks
    T = w[:, :, None] * (D / ell)
    v = linv @ ks
    return dict(mean=w.sum(0), mean_abs=np.abs(w).sum(0), J=T.sum(0), J_abs=np.abs(T).sum(0),
                var=sf2 - np.einsum('nh,nh->h', v, v), sf2=sf2)


def ks_errors(eng, X, hyper, Z, Sigma):
    """Largest normalised errors of mean / J / var of gpmpc_predict(TA) over the outputs of eng."""
    Ny = hyper.shape[0]
    mean, var, _, jac = eng.predict(Z, Sigma, L.METHOD_TA)
    e = dict(mean=0.0, J=0.0, var=0.0)
    for a in range(Ny):
        r = ks_reference(X, hyper[a], eng.get(L.GET_ALPHA, a), eng.get(L.GET_LINV, a), Z)
        e['mean'] = max(e['mean'], np.max(np.abs(mean[:, a] - r['mean']) / r['mean_abs']))
        e['J'] = max(e['J'], np.max(np.abs(jac[:, a] - r['J']) / r['J_abs']))
        e['var'] = max(e['var'], np.max(np.abs(var[:, a] - r['var'])) / r['sf2'])
    return e


@pytest.mark.parametrize('ch,Nx,Ny,N', KS_CASES)
def test_ks_chunk_buckets(ch, Nx, Ny, N):
    """Every ks_tile_kernel<NXP, CH> the dispatch reaches, at H = 50 and H = 70 (two 64-point chunks: the per-chunk
    partials are what changes with CH).  Measured on an H100 SXM: mean <= 1.1e-16 and J <= 3.3e-16 of the sum of
    |terms|, var <= 1.2e-14 of sf2.  A plain error relative to |mean| is 1e-10 here: the reference's own rounding
    (1e-16 of the sum of |terms|) over the cancellation of alpha's alternating signs.  At Nx = 32, ks_tile_kernel used
    to leave J's last 8 components of every eighth point unwritten (an error of 1e-2 of the sum of |terms|)."""
    assert ks_chunk(npad(N), Ny, Nx) == ch
    X, Y, hyper, Z, Sigma = _ks_problem(N, Nx, Ny)
    eng, info = fit(X, Y, hyper, with_info=True)
    assert not info.any()
    for H in (50, 70):
        e = ks_errors(eng, X, hyper, Z[:H], Sigma)
        assert e['mean'] < 5e-15 and e['J'] < 5e-15 and e['var'] < 1e-13, (H, e)
    eng.close()


def test_ks_chunk_1024_against_an_independent_factor():
    """CH = 1024 (Nx = 10, two outputs, the C5 headline's bucket): the full TA prediction against an independent CPU
    factor (factor_large / predict_large) at the suite's 1e-6 gate, and, at this shape, the invariants the suite checks
    below Npad 8192: gpmpc_predict_grad's values are gpmpc_predict's bits and its d var / d z matches the closed form
    on the engine's own factor; step 1 of gpmpc_rollout_sample (eps = 0) is gpmpc_predict's mean bit for bit (DESIGN
    4.12).  Measured on an H100 SXM: chol 8e-12, mean / var / J / cov <= 3.1e-10, d var / d z 2.2e-10 (the closed
    form's triangular solves carry cond(K) eps)."""
    N, Nx, Ny, H = N_KS, 10, 2, 50
    assert ks_chunk(npad(N), Ny, Nx) == 1024
    X, Y, hyper, Z, Sigma = _ks_problem(N, Nx, Ny)
    Z = Z[:H]
    eng, info = fit(X, Y, hyper, with_info=True)
    assert not info.any()
    mean, var, cov, jac = eng.predict(Z, Sigma, L.METHOD_TA)
    mo = np.zeros((H, Ny)); vo = np.zeros((H, Ny)); Jo = np.zeros((H, Ny, Nx))
    for a in range(Ny):
        f = orc.factor_large(X, Y[:, a], hyper[a])
        assert not f['jitter']
        assert relinf(eng.get(L.GET_CHOL, a), f['chol']) < 1e-9
        mo[:, a], vo[:, a], Jo[:, a] = orc.predict_large(X, hyper[a], f['alpha'], f['chol'], Z)
        del f
    co = orc.ta_cov(vo, Jo, Sigma)
    assert relinf(mean, mo) < 1e-6 and relinf(var, vo) < 1e-6 and relinf(jac, Jo) < 1e-6 and relinf(cov, co) < 1e-6
    g = eng.predict_grad(Z, Sigma, L.METHOD_TA)
    assert np.array_equal(g['mean'], mean) and np.array_equal(g['var'], var)
    assert np.array_equal(g['cov'], cov) and np.array_equal(g['jac'], jac)
    alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)])
    chol = np.stack([eng.get(L.GET_CHOL, a) for a in range(Ny)])
    cl = hso.predict_grad_closed(X, hyper, alpha, chol, Z, Sigma, 'TA')
    del chol
    assert relinf(g['dvar_dz'], cl['dvar']) < 2e-9
    mean_me = eng.predict(Z, None, L.METHOD_ME, want_cov=False, want_jac=False)[0]
    f0 = eng.rollout_sample(Z, np.repeat(Z[:, None, Ny:], 2, 1), np.zeros((H, 2, Ny)))[0][:, 0]
    assert np.array_equal(f0, mean_me)
    eng.close()


# ------------------------------------------------------------------ B. factorisation shapes and GEMM feeds
# name -> (N, outputs, small_tiles option or None, capacity or None, what the case is for)
FACTOR_CASES = {
    'n1152': (1100, 1, None, None, 'uneven split 512/640, h2 256/384'),
    'n2176': (2150, 1, None, None, 'uneven split 1024/1152, h2 512/640'),
    'n3200': (3150, 1, None, None, 'uneven split 1536/1664, h2 768/896'),
    'n1152_st0': (1100, 1, 0, None, 'no 64x32: gemm_dmma_kernel<128,64,...,true,...> on the deep levels'),
    'n2176_st0': (2150, 1, 0, None, 'no 64x32'),
    'n3200_st0': (3150, 1, 0, None, 'no 64x32'),
    'n1152_all64': (1100, 1, 1 << 30, None, 'every product on 64x32'),
    'n2176_all64': (2150, 1, 1 << 30, None, 'every product on 64x32'),
    'n3200_all64': (3150, 1, 1 << 30, None, 'every product on 64x32'),
    'n4224x3': (4200, 3, None, None, 'TMA panels on uneven splits'),
    'n1152x24': (1130, 24, None, None, 'TMA at small N through the batch'),
    'n2176x12': (2100, 12, None, None, 'TMA at small N through the batch'),
    'n4096x8': (4000, 8, None, None, 'TMA SYRK in lower mode with batch > 1'),
    'reserve2176': (1900, 2, None, 2100, 'reserved handle, Npad 2176: uneven split'),
}
# what each TMA case must reach on the device at hand (checked through factor_feeds)
TMA_TARGET = {'n4224x3': lambda f: any(s == 'panel' and fd == 'tma' and n1 != n2 for s, fd, _, _, n1, n2, _ in f),
              'n1152x24': lambda f: any(fd == 'tma' for _, fd, *_ in f),
              'n2176x12': lambda f: any(fd == 'tma' for _, fd, *_ in f),
              'n4096x8': lambda f: any(fd == 'tma' and lw for _, fd, _, lw, *_ in f)}
# (chol, L^-1, alpha, logdet) bars relative to the LAPACK factor of the engine's K: the synthetic problem (sn = 1e-2,
# cond K up to ~1e8) and the well-conditioned variant (sn = 0.3)
FACTOR_TOL = {'sn1e-2': (1e-10, 1e-9, 1e-7, 1e-12), 'sn0.3': (2e-13, 1e-12, 4e-12, 1e-14)}


def _factor_problem(N, Ny, cond):
    p = orc.synthetic_problem(N, 6, Ny, config_id=200 + Ny)
    hyper = p['hyper'].copy()
    if cond == 'sn0.3':
        hyper[:, -1] = 0.3
    return p['X'], p['Y'], hyper


def factor_errors(eng, Y):
    """Largest errors over the outputs of eng against LAPACK on the engine's own K."""
    N = eng.N
    e = dict(chol=0.0, linv=0.0, linv_l=0.0, alpha=0.0, logdet=0.0)
    for a in range(eng.out_count):
        K = eng.get(L.GET_K, a)
        Lc = np.linalg.cholesky(K)
        del K
        chol = eng.get(L.GET_CHOL, a)
        linv = eng.get(L.GET_LINV, a)
        e['chol'] = max(e['chol'], relinf(chol, Lc))
        e['linv'] = max(e['linv'], relinf(linv, solve_triangular(Lc, np.eye(N), lower=True, check_finite=False)))
        e['linv_l'] = max(e['linv_l'], np.abs(linv @ chol - np.eye(N)).max())
        e['alpha'] = max(e['alpha'], relinf(eng.get(L.GET_ALPHA, a), cho_solve((Lc, True), Y[:, a], check_finite=False)))
        ld = 2 * np.sum(np.log(np.diag(Lc)))
        e['logdet'] = max(e['logdet'], abs(eng.get(L.GET_LOGDET, a)[0] - ld) / abs(ld))
    return e


def _factor_engine(name, cond):
    N, Ny, st, cap, _ = FACTOR_CASES[name]
    X, Y, hyper = _factor_problem(N, Ny, cond)
    import gp_mpc_b200
    eng = gp_mpc_b200.Engine(N, X.shape[1], Ny, device=0, capacity=cap)
    if st is not None:
        eng.set_option('small_tiles', st)
    eng.set_data(X, Y); eng.set_hyper(hyper)
    return eng, Y


@pytest.mark.parametrize('cond', ['sn1e-2', 'sn0.3'])
@pytest.mark.parametrize('name', list(FACTOR_CASES))
def test_factorisation_against_lapack(name, cond):
    """L, L^-1, alpha and log det of every output against LAPACK on the engine's K.  Measured on an H100 SXM, largest
    over the cases: sn = 1e-2: chol 6.4e-12, L^-1 1.0e-10, L^-1 L - I 9.3e-13, alpha 9.8e-10, logdet 8.7e-14 (cond(K) eps;
    chol and alpha keep the suite's bars 1e-10 and 1e-7); sn = 0.3: chol 2.5e-14, L^-1 8.6e-14, L^-1 L - I 7.5e-15,
    alpha 3.9e-13, logdet 5.9e-16.  A (1 + 1e-9) factor in any GEMM's epilogue moves L by about 1e-9.
    Factorising again gives the same bits: every GEMM element and leaf has a fixed order, so a difference is a race
    between the look-ahead side streams and the main stream."""
    N, Ny, st, cap, _ = FACTOR_CASES[name]
    if name in TMA_TARGET:
        require(TMA_TARGET[name](factor_feeds(npad(max(N, cap or 0)), Ny, sms(), st)), 'the TMA feed')
    eng, Y = _factor_engine(name, cond)
    info = eng.factorize()
    assert not info.any()
    e = factor_errors(eng, Y)
    tc, tl, ta, td = FACTOR_TOL[cond]
    assert e['chol'] < tc and e['linv'] < tl and e['linv_l'] < tl and e['alpha'] < ta and e['logdet'] < td, e
    first = [(eng.get(L.GET_CHOL, a), eng.get(L.GET_LINV, a), eng.get(L.GET_ALPHA, a)) for a in range(Ny)]
    eng.factorize()
    for a in range(Ny):
        again = (eng.get(L.GET_CHOL, a), eng.get(L.GET_LINV, a), eng.get(L.GET_ALPHA, a))
        for x, y in zip(first[a], again):
            assert np.array_equal(x, y), a
    eng.close()


def _factors(eng):
    return [np.stack([eng.get(w, a) for a in range(eng.out_count)]) for w in (L.GET_CHOL, L.GET_LINV, L.GET_ALPHA)]


@pytest.mark.parametrize('n', ['n1152', 'n2176', 'n3200'])
def test_cp_async_feeds_agree_bit_for_bit(n):
    """The 64x32 and 128x64 cp.async GEMMs give the same bits: each element's k order is the same and the larger
    tile's extra k-steps multiply exact zeros (measured: identical at 1152, 2176 and 3200 rows).  The default mix of
    the two equals both."""
    outs = []
    for name in (n, n + '_st0', n + '_all64'):
        eng, _ = _factor_engine(name, 'sn1e-2')
        eng.factorize()
        outs.append(_factors(eng))
        eng.close()
    for other in outs[1:]:
        for x, y in zip(outs[0], other):
            assert np.array_equal(x, y)


def test_tma_feed_agrees_with_cp_async():
    """The TMA tensor-map GEMM against the same factorisation with every product on 64x32 tiles (small_tiles = 2^30),
    at 4096 x 8 outputs, where the lower-mode SYRK updates run on TMA.  The two do not give the same bits (the TMA
    kernel sums each element's k-steps in another order); measured on an H100 SXM: chol 3.3e-12, L^-1 6.1e-11, alpha
    1.3e-10 apart, the cond(K) eps of this problem."""
    require(TMA_TARGET['n4096x8'](factor_feeds(4096, 8, sms())), 'the TMA feed')
    outs = []
    for st in (None, 1 << 30):
        eng, _ = _factor_engine('n4096x8', 'sn1e-2')
        if st is not None:
            eng.set_option('small_tiles', st)
        eng.factorize()
        outs.append(_factors(eng))
        eng.close()
    for x, y, tol in zip(*outs, (3e-11, 6e-10, 1.3e-9)):
        assert relinf(x, y) < tol


def test_jitter_rerun_of_one_output_in_a_batch():
    """factor_entries' lone reruns of a failed output (zero jitter, then 1e-8) on a split shape: one of three outputs at
    Npad 1152 has duplicated points and sn = 1e-10, so its K is singular in fp64.  Its info is 1 and its factor is LAPACK's of
    K + 1e-8 I (measured 8e-10; cond ~1e11); the other two outputs hold the bits of a batch without the singular
    output."""
    N, Nx = 1100, 6
    p = orc.synthetic_problem(N, Nx, 3, config_id=301)
    X = p['X'].copy(); X[N // 2:] = X[:N - N // 2]
    bad = p['hyper'].copy(); bad[1, Nx + 1] = 1e-10
    eng, info = fit(X, p['Y'], bad, with_info=True)
    assert list(info) == [0, 1, 0]
    K = eng.get(L.GET_K, 1) + 1e-8 * np.eye(N)
    assert relinf(eng.get(L.GET_CHOL, 1), np.linalg.cholesky(K)) < 1e-8
    ref, info_r = fit(X, p['Y'], p['hyper'], with_info=True)
    assert not info_r.any()
    for a in (0, 2):
        for w in (L.GET_CHOL, L.GET_LINV, L.GET_ALPHA):
            assert np.array_equal(eng.get(w, a), ref.get(w, a))
    eng.close(); ref.close()


# ------------------------------------------------------------------ C. NLML value and gradient, K^-1
NLML_CASES = [(300, 3), (300, 12), (300, 17), (300, 32), (1100, 12), (3000, 5)]


def nlml_grad_reference(th, X, y):
    """dNLL/dtheta (R&W eq. 5.9, the parametrisation of calc_NLL_grad_analytic) and the sum of |terms| of each
    component, with K^-1 from LAPACK."""
    n, D = X.shape
    ell = th[:D]; sf = th[D]; sn = th[D + 1]
    Kf = orc.covSEard(X, X, ell, sf ** 2)
    Lc = np.linalg.cholesky(Kf + sn ** 2 * np.eye(n))
    Kinv = cho_solve((Lc, True), np.eye(n), check_finite=False)
    alpha = cho_solve((Lc, True), y, check_finite=False)
    WK = (Kinv - np.outer(alpha, alpha)) * Kf
    g = np.zeros(D + 2); s = np.zeros(D + 2)
    for d in range(D):
        t = WK * (X[:, d][:, None] - X[:, d][None, :]) ** 2
        g[d] = 0.5 * t.sum() / ell[d] ** 3
        s[d] = 0.5 * np.abs(t).sum() / ell[d] ** 3
    g[D] = WK.sum() / sf; s[D] = np.abs(WK).sum() / sf
    w = np.diag(Kinv) - alpha * alpha
    g[D + 1] = w.sum() * sn; s[D + 1] = np.abs(w).sum() * sn
    return g, s


def _nlml_theta(hyper_a, cond):
    th = hyper_a.copy()
    Nx = th.size - 2
    th[:Nx] *= 0.8
    th[Nx + 1] = 1e-2 if cond == 'ill' else 0.3
    return th


def nlml_errors(N, Nx, cond):
    p = orc.synthetic_problem(N, Nx, 1, config_id=400 + Nx)
    X, y = p['X'], p['Y'][:, 0]
    import gp_mpc_b200
    eng = gp_mpc_b200.Engine(N, Nx, 1, device=0)
    eng.set_data(X, p['Y'])
    th = _nlml_theta(p['hyper'][0], cond)
    nll, g = eng.nlml(0, th, grad=True)
    eng.close()
    gr, s = nlml_grad_reference(th, X, y)
    return dict(nll=abs(nll - orc.calc_NLL(th, X, y)) / abs(orc.calc_NLL(th, X, y)),
                grad=np.max(np.abs(g - gr) / s), grad_rel=relinf(g, gr))


# (nll, gradient / sum of |terms|): at sn = 1e-2, K^-1 (the reference's own too) is cond(K) eps-limited and calc_NLL's
# expansion-form K moves the NLL by 1e-11 relative to the direct differences at Nx = 3
NLML_TOL = {'ill': (1e-10, 1e-8), 'well': (1e-13, 4e-14)}


@pytest.mark.parametrize('cond', ['ill', 'well'])
@pytest.mark.parametrize('N,Nx', NLML_CASES)
def test_nlml_value_and_gradient(N, Nx, cond):
    """nlml_grad_kernel<8 / 16 / 32> (Nx 3, 12, 17, 32 at N = 300), Nx = 12 at N = 1100 (uneven split, a partial 64-tile
    of the gradient kernel) and Nx = 5 at N = 3000 (kinv_at's SYRK on the TMA feed).  Measured on an H100 SXM:
    sn = 1e-2: nll <= 8.1e-12, gradient <= 5.3e-14 of the sum of |terms| (the gradient keeps the suite's 1e-8 bar);
    sn = 0.3: nll <= 3.3e-15, gradient <= 4.0e-15."""
    if N == 3000:
        require(gemm_feed(24, 24, 1, True, 1, sms())[0] == 'tma', 'the TMA feed')
    e = nlml_errors(N, Nx, cond)
    tn, tg = NLML_TOL[cond]
    assert e['nll'] < tn and e['grad'] < tg, e


@pytest.mark.parametrize('cond', ['ill', 'well'])
def test_invk_against_lapack_on_the_tma_feed(cond):
    """GET_INVK at N = 3000 (Npad 3072: compute_kinv's U U^T runs on the TMA kernel with the GE k-flags, in kinv_at)
    against the LAPACK inverse of the engine's K.  Measured on an H100 SXM: sn = 1e-2 9.1e-11 (cond(K) eps), sn = 0.3
    6.6e-14."""
    require(gemm_feed(24, 24, 1, True, 1, sms())[0] == 'tma', 'the TMA feed')
    N, Nx = 3000, 5
    p = orc.synthetic_problem(N, Nx, 1, config_id=400 + Nx)
    hyper = _nlml_theta(p['hyper'][0], cond)[None, :]
    eng, info = fit(p['X'], p['Y'], hyper, with_info=True)
    assert not info.any()
    K = eng.get(L.GET_K, 0)
    ref = cho_solve((np.linalg.cholesky(K), True), np.eye(N), check_finite=False)
    invk = eng.get(L.GET_INVK, 0)
    assert np.array_equal(invk, invk.T)
    assert relinf(invk, ref) < (1e-8 if cond == 'ill' else 1e-12)
    eng.close()

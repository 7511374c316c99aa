"""gpmpc_nlml_batch and multi-start fits ('starts': 'lhs') on the GPU: every entry bit-identical to gpmpc_nlml whatever
the batch, its order and the pass size; agreement with the oracle; NOTPD entries; the factorisation left as it was; the
argument and state checks; and end-to-end fits on the fixtures and on a data set with two optima."""
import ctypes as C
import re

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._util import GOLDEN, load_fixture, relinf

pytestmark = pytest.mark.gpu


def _engine(X, Y, **kw):
    eng = L.Engine(X.shape[0], X.shape[1], Y.shape[1], device=0, **kw)
    eng.set_data(X, Y)
    return eng


def _thetas(hyper_row, n, seed):
    """n hyper rows around hyper_row: length scales and sf within a factor 2, sn in [1e-3, 1e-2]."""
    rng = np.random.default_rng(seed)
    d = hyper_row.size
    th = np.tile(hyper_row, (n, 1))
    th[:, :d - 1] *= 2.0 ** rng.uniform(-1, 1, (n, d - 1))
    th[:, d - 1] = 10.0 ** rng.uniform(-3, -2, n)
    return th


# N, Nx: nlml_grad_kernel<8 / 16 / 32>.  With the feed chosen per slab, every size takes the 64x32 feed on its small
# products, Npad 4096 the TMA feed on its NT products with 528 or more tiles, and Npad 4352 also the 128x64 cp.async feed
# on its top-level NN products (2 * 17 * 17 tiles)
@pytest.mark.parametrize('N,Nx', [(300, 3), (1100, 12), (4096, 32), (4352, 8)])
def test_every_entry_is_bit_identical_to_nlml(N, Nx):
    p = orc.synthetic_problem(N, Nx, 2, config_id=N + Nx)
    eng = _engine(p['X'], p['Y'])
    a = 1
    th = _thetas(p['hyper'][a], 8, N)
    ref = [eng.nlml(a, t, grad=True) for t in th]
    ref_nog = [eng.nlml(a, t, grad=False) for t in th]
    for rows in ([6], [4, 1, 4], [5, 2, 2, 7, 0, 1, 5, 3]):          # S = 1, 3, 8: shuffled and duplicated
        for cap in (0, 1, 3):
            eng.set_option('nlml_batch_max', cap)
            nll, g, st = eng.nlml_batch(a, th[rows], grad=True)
            assert not st.any()
            for i, r in enumerate(rows):
                assert nll[i] == ref[r][0] and np.array_equal(g[i], ref[r][1]), (rows, cap, i)
            nll, g, st = eng.nlml_batch(a, th[rows], grad=False)
            assert g is None and not st.any()
            assert all(nll[i] == ref_nog[r] for i, r in enumerate(rows)), (rows, cap)
    eng.close()


# (NLL relative, gradient relinf): tank's K has cond ~1e7 at these rows, as test_nlml_gradient_vs_oracle's problem, and
# gets its bars; car's reaches cond ~1e9-1e10 on the raw fixture, and both errors carry cond(K) eps
ORACLE_TOL = {'tank': (1e-10, 1e-8), 'car': (1e-8, 1e-5)}


@pytest.mark.parametrize('case', ['tank', 'car'])
def test_agrees_with_the_oracle_on_the_fixtures(case):
    m = load_fixture(case)
    X, Y = m['X'], m['Y']
    Nx = X.shape[1]
    eng = _engine(X, Y)
    for a in range(Y.shape[1]):
        th = np.tile(m['hyper'][a, :Nx + 2], (3, 1))
        th[:, :Nx] *= np.array([0.5, 1.0, 2.0])[:, None]
        th[:, Nx + 1] = 5e-3
        nll, g, st = eng.nlml_batch(a, th)
        assert not st.any()
        for s in range(3):
            assert nll[s] == pytest.approx(orc.calc_NLL(th[s], X, Y[:, a]), rel=ORACLE_TOL[case][0])
            assert relinf(g[s], orc.calc_NLL_grad_analytic(th[s], X, Y[:, a])) < ORACLE_TOL[case][1]
    eng.close()


def test_a_notpd_entry_leaves_the_others_and_reports_what_nlml_reports():
    p = orc.synthetic_problem(300, 4, 1, config_id=9)
    X = p['X'].copy()
    X[150:] = X[:150]                         # every point twice: at sn = 1e-10 K is singular to rounding
    Y = p['Y'].copy()
    Y[150:] = Y[:150]
    eng = _engine(X, Y)
    good = _thetas(p['hyper'][0], 3, 1)
    dup = p['hyper'][0].copy()
    dup[-1] = 1e-10
    nan = good[0].copy()
    nan[4] = np.nan                           # a NaN signal std fails every pivot, with and without the jitter
    th = np.vstack([good[0], nan, good[1], dup, good[2]])
    nll, g, st = eng.nlml_batch(0, th)
    assert st[1] == L.ERR_NOTPD and np.isnan(nll[1]) and np.isnan(g[1]).all()
    alone_nll, alone_g, _ = eng.nlml_batch(0, good)
    for i, s in ((0, 0), (2, 1), (4, 2)):
        assert st[i] == 0 and nll[i] == alone_nll[s] and np.array_equal(g[i], alone_g[s])
    for i in range(len(th)):
        # status against nlml's outcome and against factorize's jitter report at the same row
        hyp = th[i:i + 1]
        if st[i] == L.ERR_NOTPD:
            with pytest.raises(np.linalg.LinAlgError):
                eng.nlml(0, th[i])
            eng.set_hyper(hyp)
            with pytest.raises(np.linalg.LinAlgError):
                eng.factorize()
        else:
            f, gr = eng.nlml(0, th[i])
            assert f == nll[i] and np.array_equal(gr, g[i])
            eng.set_hyper(hyp)
            assert eng.factorize()[0] == st[i]
    eng.close()


def test_the_factorisation_is_left_as_it_was():
    p = orc.synthetic_problem(700, 5, 3, config_id=21)
    eng = _engine(p['X'], p['Y'])
    eng.set_hyper(p['hyper'])
    eng.factorize()
    Z = np.random.default_rng(0).standard_normal((20, 5))

    def state():
        out = list(eng.predict(Z, 1e-3 * np.eye(5))) + list(eng.loo())
        for a in range(3):
            out += [eng.get(w, a) for w in (L.GET_CHOL, L.GET_ALPHA, L.GET_LINV)]
        return out

    before = state()
    for a in range(3):
        eng.nlml_batch(a, _thetas(p['hyper'][a], 4, a))
    for x, y in zip(before, state()):
        assert np.array_equal(x, y)
    eng.close()


def test_argument_and_state_errors_come_before_any_work():
    p = orc.synthetic_problem(200, 3, 2, config_id=3)
    th = _thetas(p['hyper'][0], 3, 0)
    eng = L.Engine(200, 3, 2, out_begin=1, out_count=1, device=0)
    nll = np.full(3, 7.0)
    st = np.zeros(3, dtype=np.int32)
    ptr = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
    sp = st.ctypes.data_as(C.POINTER(C.c_int))
    assert L.load().gpmpc_nlml_batch(eng.h, 1, 3, ptr(th), ptr(nll), None, sp) == L.ERR_STATE     # no data
    eng.set_data(p['X'], p['Y'])
    zero = th.copy()
    zero[2, 1] = 0.0
    for a, S, t, n, s in ((1, 0, th, nll, sp), (1, 3, None, nll, sp), (1, 3, th, None, sp), (1, 3, th, nll, None),
                          (0, 3, th, nll, sp), (1, 3, zero, nll, sp)):
        rc = L.load().gpmpc_nlml_batch(eng.h, a, S, None if t is None else ptr(t), None if n is None else ptr(n), None, s)
        assert rc == L.ERR_ARG, (a, S)
        assert (nll == 7.0).all()
    with pytest.raises(L.GpmpcError):
        eng.set_option('nlml_batch_max', -1)
    eng.close()


def _states(out):
    """{output: winning start} from train_gp_b200's verbose lines."""
    return {int(a): int(s) for a, s in re.findall(r'\* State (\d+):.*start (\d+) of', out)}


@pytest.mark.parametrize('case', ['tank', 'car'])
def test_fixture_fits_never_get_worse_and_repeat_bit_for_bit(case, capsys):
    import gp_mpc_b200
    m = load_fixture(case)
    opts = {'starts': 'lhs'}
    one = gp_mpc_b200.GP(m['X'], m['Y'])
    capsys.readouterr()
    four = gp_mpc_b200.GP(m['X'], m['Y'], multistart=4, optimizer_opts=opts)
    win = _states(capsys.readouterr().out)
    again = gp_mpc_b200.GP(m['X'], m['Y'], multistart=4, optimizer_opts=opts)
    h1, h4 = one._GP__hyper, four._GP__hyper
    assert np.array_equal(h4, again._GP__hyper)
    assert sorted(win) == list(range(m['Y'].shape[1]))
    eng = four.engine
    for a in range(m['Y'].shape[1]):
        if win[a] == 0:
            assert np.array_equal(h4[a], h1[a])
        assert eng.nlml(a, h4[a], grad=False) <= eng.nlml(a, h1[a], grad=False)


def test_two_optima_data_set_improves_strictly():
    from gp_mpc_b200.optimize import train_gp_b200
    z = np.load(GOLDEN + '/multistart_two_optima.npz')
    X, Y = z['X'], z['Y']
    eng = _engine(X, Y)
    one = train_gp_b200(eng, X, Y, verbose=False)[0]
    four = train_gp_b200(eng, X, Y, multistart=4, optimizer_opts={'starts': 'lhs'}, verbose=False)[0]
    f1, f4 = eng.nlml(0, one, grad=False), eng.nlml(0, four, grad=False)
    assert f4 < f1 - 1.0, (f1, f4)
    eng.close()

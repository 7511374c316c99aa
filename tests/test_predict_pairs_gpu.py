"""The predict product's paired schedule (predict_streamk.cuh, psk_pair_units) at 8 outputs on one H100: N = 16384 (the
C5 shape: 64 tiles, 256 units), 8320 (Npad / 128 odd: the pair holding the half tile is 8 steps shorter) and 8448 (33
tiles: the middle tile is a unit alone).  The last two have 136 units, which the automatic 132-CTA grid would run in two
half-filled rounds, so they stay on stream-K there and run paired here on 68 CTAs (predict_ctas).  var matches
sf2 - |L^-1 ks|^2 formed in long double, with the bar of test_predict_panel_gpu; and because no tile is cut, var is bitwise
the same on every grid that pairs (N = 16384: the automatic 128 CTAs of psk_pair_grid, 64 and 132; else 68, 34 and 136),
for a point in any row of an H = 1, 8 or 50 batch, and from predict_grad, whose product also stores the solved rows."""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._util import PREDICT_VAR_TOL

pytestmark = pytest.mark.gpu

LD = np.longdouble
NX, NY, H = 10, 8, 50
SIZES = (8320, 8448, 16384)
GRIDS = {16384: (0, 64, 132), 8320: (68, 34, 136), 8448: (68, 34, 136)}      # first: the grid of the other tests


@pytest.fixture(scope='module', params=SIZES)
def model(request):
    N = request.param
    p = orc.synthetic_problem(N, NX, NY, config_id=900 + N % 97, H=H)
    eng = L.Engine(N, NX, NY, device=0)
    eng.set_data(p['X'], p['Y'])
    eng.set_hyper(p['hyper'])
    assert not eng.factorize().any()
    eng.set_option('predict_ctas', GRIDS[N][0])
    yield N, eng, p
    eng.close()


def predict_var(eng, Z, Sigma):
    return eng.predict(Z, Sigma, L.METHOD_TA, want_cov=False, want_jac=False)[1]


def test_var_matches_long_double_linv_ks(model):
    N, eng, p = model
    X, hyper = p['X'], p['hyper']
    var = predict_var(eng, p['Z'], p['Sigma'])
    rows = [0, H - 1]                                  # first and last row of the 56-row chunk
    Z = p['Z'][rows].astype(LD)
    worst = 0.0
    for a in range(NY):
        ell, sf2 = LD(1) * hyper[a, :NX], LD(hyper[a, NX]) ** 2
        d = (X.astype(LD)[:, None, :] - Z[None, :, :]) / ell
        ks = sf2 * np.exp(-0.5 * np.sum(d * d, axis=2))                  # (N, 2)
        Li = eng.get(L.GET_LINV, a)
        v, w = np.zeros((N, len(rows)), LD), np.zeros((N, len(rows)), LD)
        for r0 in range(0, N, 2048):                                   # L^-1 is lower triangular
            r1 = min(N, r0 + 2048)
            blk = Li[r0:r1, :r1].astype(LD)
            v[r0:r1], w[r0:r1] = blk @ ks[:r1], np.abs(blk) @ ks[:r1]
        del Li
        ref, scale = sf2 - np.sum(v * v, axis=0), sf2 + np.sum(w * w, axis=0)
        err = float(np.max(np.abs(var[rows, a].astype(LD) - ref) / scale))
        worst = max(worst, err)
        assert err <= PREDICT_VAR_TOL, (N, a, err)
    print('MEASURED N=%d var vs long double %.2e' % (N, worst))


def test_var_does_not_depend_on_the_grid(model):
    N, eng, p = model
    ref = predict_var(eng, p['Z'], p['Sigma'])
    try:
        for ctas in GRIDS[N][1:]:
            eng.set_option('predict_ctas', ctas)
            assert np.array_equal(predict_var(eng, p['Z'], p['Sigma']), ref), (N, ctas)
    finally:
        eng.set_option('predict_ctas', GRIDS[N][0])


def test_var_does_not_depend_on_batch_or_row(model):
    N, eng, p = model
    Z, S = p['Z'], p['Sigma']
    ref = predict_var(eng, Z, S)
    rng = np.random.default_rng(N)
    for Hb in (1, 8, 50):
        idx = rng.permutation(H)[:Hb]
        assert np.array_equal(predict_var(eng, Z[idx], S), ref[idx]), (N, Hb)


def test_predict_grad_product_repeats_the_fused_var(model):
    """predict_grad's first product stores the solved rows (Vout) next to the records: the same schedule, the same var.
    Not at N = 16384, where its second operand U = L^-T would add 17 GB for 8 outputs."""
    N, eng, p = model
    if N == 16384:
        pytest.skip('U = L^-T of 8 outputs at N = 16384 does not fit next to the predict buffers')
    Z = p['Z'][:8]
    g = eng.predict_grad(Z, p['Sigma'], L.METHOD_TA)
    assert np.array_equal(g['var'], predict_var(eng, Z, p['Sigma']))

"""GP.append_data under a prior mean function on CPU, through the oracle-backed engine: the rank-1 appends hand the
engine the residual y - m(x), the targets the factorisation uses, so the model equals a GP built on all points, whether
or not the refit fallback fired in an earlier call."""
import numpy as np
import pytest

import gp_mpc_b200
from gp_mpc_b200 import mean_functions as mf
from oracle import gp_oracle as orc
from tests._fake_engine import OracleEngine
from tests._util import relinf

N, NX, NY = 30, 3, 2


def _problem(func):
    p = orc.synthetic_problem(N, NX, NY, config_id=21)
    hyper = np.hstack([p['hyper'], 0.5 * np.random.default_rng(4).standard_normal((NY, mf.count_mean_params(func, NX)))])
    return p['X'], p['Y'], hyper


def _meta():
    """Standardisation of a caller whose data are X * stdZ + meanZ, Y * stdY + meanY (the GP keeps X, Y standardised)."""
    meanZ, stdZ = np.array([0.3, -1.0, 2.0]), np.array([1.5, 0.7, 2.0])
    return dict(meanY=np.array([1.0, -2.0]), stdY=np.array([0.5, 3.0]), meanZ=meanZ, stdZ=stdZ,
                meanX=meanZ[:NY], stdX=stdZ[:NY], meanU=meanZ[NY:], stdU=stdZ[NY:])


def _gp(X, Y, hyper, func, meta):
    kw = dict(meta=meta) if meta is not None else {}
    return gp_mpc_b200.GP(X, Y, mean_func=func, hyper=dict(hyper=hyper), normalize=meta is not None,
                          engine_factory=OracleEngine, **kw)


def _caller_units(X, Y, meta):
    if meta is None:
        return X, Y
    return X * meta['stdZ'] + meta['meanZ'], Y * meta['stdY'] + meta['meanY']


def _assert_same_model(gp, ref):
    assert gp.get_size()[0] == ref.get_size()[0] == N
    assert relinf(gp.get_chol(), ref.get_chol()) < 1e-10
    assert relinf(gp.get_alpha(), ref.get_alpha()) < 1e-10


@pytest.mark.parametrize('func,normalize', [('const', False), ('linear', False), ('linear', True)])
def test_append_data_under_a_prior_mean_equals_a_gp_on_all_points(func, normalize):
    X, Y, hyper = _problem(func)
    meta = _meta() if normalize else None
    gp = _gp(X[:N - 3], Y[:N - 3], hyper, func, meta)
    eng = gp.engine
    gp.append_data(*_caller_units(X[N - 3:], Y[N - 3:], meta))
    assert gp.engine is eng                               # rank-1 appends, no refit
    _assert_same_model(gp, _gp(X, Y, hyper, func, meta))


def test_appends_after_a_refit_fallback_equal_a_gp_on_all_points(monkeypatch):
    X, Y, hyper = _problem('linear')
    gp = _gp(X[:N - 4], Y[:N - 4], hyper, 'linear', None)
    eng = gp.engine
    # the second append of the first call loses positive definiteness: that call ends in a refit on all its points
    monkeypatch.setattr(OracleEngine, 'fail_on', (0, N - 3))
    gp.append_data(X[N - 4:N - 2], Y[N - 4:N - 2])
    assert gp.engine is not eng and gp.get_size()[0] == N - 2
    refit = gp.engine
    gp.append_data(X[N - 2:], Y[N - 2:])                  # rank-1 appends on the refitted engine
    assert gp.engine is refit
    _assert_same_model(gp, _gp(X, Y, hyper, 'linear', None))

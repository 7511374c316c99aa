"""Host-side behaviour of the GP class (constructor paths, standardisation quirks, JSON schema,
error types, mean-function bookkeeping) exercised on CPU through the oracle-backed stand-in
engine (tests/_fake_engine.py).  The arithmetic itself is covered by the -m gpu tests."""
import json

import numpy as np
import pytest

import gp_mpc_b200
from oracle import gp_oracle as orc
from tests._fake_engine import OracleEngine, OracleEngineWithRollout, fixture_gp
from tests._util import load_golden, relinf


def _gp(name, **kw):
    return fixture_gp(name, OracleEngine, **kw)


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_predict_wrapper_follows_the_reference(name):
    """gp_class.py:245-263: x,u standardised, mean de-standardised, covariance NOT rescaled."""
    gp, m = _gp(name)
    d = load_golden('derived', name)
    tol = 1e-8 if name == 'tank' else 1e-6       # car: cond(K) ~ 1e10, factors are recomputed from (X, hyper)
    mean, cov = gp.predict(d['x0'], d['u0'], d['Sigma'])
    assert relinf(mean, d['mean_ta']) < tol and relinf(cov, d['cov_ta']) < tol
    assert mean.shape == (m['Y'].shape[1], 1)
    gp.set_method('ME')
    mean, cov = gp.predict(d['x0'], d['u0'], None)
    assert relinf(cov, d['cov_me']) < tol
    A, B = gp.discrete_linearize(d['x0'], d['u0'], d['Sigma'])
    assert relinf(A, d['A']) < tol and relinf(B, d['B']) < tol
    with pytest.raises(NameError):
        gp.set_method('XY')
    with pytest.raises(NotImplementedError):
        gp.set_method('old_ME')


def test_json_schema_and_hyper_views(tmp_path):
    gp, m = _gp('tank')
    hp = gp.get_hyper_parameters()
    assert np.array_equal(hp['length_scale'], m['hyper'][:, :6])
    assert np.allclose(hp['signal_var'], m['signal_var']) and np.allclose(hp['noise_var'], m['noise_var'])
    assert np.array_equal(hp['mean'], m['hyper'][:, 7:])            # includes sn as first column (q1)
    gp.save_model(str(tmp_path / 'mdl'))
    dd = json.load(open(str(tmp_path / 'mdl') + '.json'))
    assert set(dd) == {'X', 'Y', 'hyper', 'mean_func', 'normalize', 'xlb', 'xub', 'ulb', 'uub', 'meta'}
    assert set(dd['meta']) == {'meanY', 'stdY', 'meanZ', 'stdZ', 'meanX', 'stdX', 'meanU', 'stdU'}
    assert np.array_equal(np.array(dd['X']), m['X'])                # stored standardised, not re-standardised
    gp2 = gp_mpc_b200.GP.load_model(str(tmp_path / 'mdl'), engine_factory=OracleEngine)
    assert gp2.get_size() == gp.get_size() == (60, 4, 2)


def test_training_statistics_and_mean_function_bookkeeping():
    p = orc.synthetic_problem(30, 3, 2, config_id=9)
    Xr = 5.0 + 2.0 * p['X']; Yr = -1.0 + 0.3 * p['Y']
    gp = gp_mpc_b200.GP(Xr, Yr, normalize=True, xlb=[0, 0], xub=[1, 1], ulb=[0], uub=[1], mean_func='linear',
                        optimizer_opts={'maxiter': 20}, engine_factory=OracleEngine)
    # 'linear' adds Nx+1 mean parameters per output that the numeric path leaves at zero
    hp = gp.get_hyper_parameters()
    assert hp['mean'].shape == (2, 1 + 3 + 1) and np.all(hp['mean'][:, 1:] == 0.0)
    st = orc.data_stats(Xr, Yr, 2)
    d = gp._GP__to_dict()
    for k in st:
        assert np.allclose(d['meta'][k], st[k])
    assert np.allclose(np.array(d['X']), (Xr - st['meanZ']) / st['stdZ'])
    with pytest.raises(NameError):
        gp_mpc_b200.GP(Xr, Yr, mean_func='cubic', engine_factory=OracleEngine, xlb=[0, 0], xub=[1, 1], ulb=[0], uub=[1])
    with pytest.raises(ValueError):
        gp_mpc_b200.GP(Xr, Yr[:-1], engine_factory=OracleEngine)


def test_validate_matches_oracle_and_prints_banners(capsys):
    gp, m = _gp('tank')
    rng = np.random.default_rng(3)
    Xt = m['meta']['meanZ'] + m['meta']['stdZ'] * rng.standard_normal((15, 6)) * 0.4
    Yt = m['meta']['meanY'] + m['meta']['stdY'] * rng.standard_normal((15, 4)) * 0.4
    smse, mnlp = gp.validate(Xt, Yt)
    so, mo = orc.validate(dict(m, alpha=gp.get_alpha(), chol=gp.get_chol()), Xt, Yt)
    assert relinf(smse, so) < 1e-9 and relinf(mnlp, mo) < 1e-9
    out = capsys.readouterr().out
    assert '# Validation of GP model' in out and '* Standardized mean squared error:' in out
    gp.print_hyper_parameters()
    assert '# Hyper-parameters' in capsys.readouterr().out


def test_prior_mean_functions_follow_the_reference():
    """get_mean_function (gp_functions.py:25-69): parameter layout at the tail of the hyper row,
    alpha on the residual y - m(X) (optimize.py:492-494), prediction without m(z) by default (q2)
    and with it under the flag.  Host logic only: the engine is the oracle-backed stand-in."""
    import gp_mpc_b200
    from gp_mpc_b200 import mean_functions as mf
    from tests._fake_engine import OracleEngine, OracleEngineWithRollout
    rng = np.random.default_rng(2)
    p = orc.synthetic_problem(30, 3, 2, config_id=21, H=5)
    Nx = 3
    for func, h_m in (('const', 1), ('linear', Nx + 1), ('polynomial', 2 * Nx + 1)):
        assert mf.count_mean_params(func, Nx) == h_m
        hyper = np.hstack([p['hyper'], 0.3 * rng.standard_normal((2, h_m))])
        for a in range(2):
            m_ref = orc.mean_function(hyper[a], p['X'], func)
            np.testing.assert_allclose(mf.mean_function(hyper[a], p['X'], func), m_ref, rtol=1e-13, atol=1e-14)
            np.testing.assert_allclose(mf.mean_design(p['X'], func) @ hyper[a, Nx + 2:], m_ref, rtol=1e-13, atol=1e-14)
            # Jacobian of the mean vs central differences
            Jm = mf.mean_jacobian(hyper[a], p['Z'], func)
            for d in range(Nx):
                e = np.zeros(Nx); e[d] = 1e-6
                fd = (mf.mean_function(hyper[a], p['Z'] + e, func) - mf.mean_function(hyper[a], p['Z'] - e, func)) / 2e-6
                np.testing.assert_allclose(Jm[:, d], fd, rtol=1e-6, atol=1e-8)
        post = orc.postfit(p['X'], p['Y'], hyper, lapack_general_solve=False, mean_func=func)
        kw = dict(hyper=dict(hyper=hyper), normalize=False, mean_func=func, engine_factory=OracleEngine)
        gp = gp_mpc_b200.GP(p['X'], p['Y'], **kw)
        np.testing.assert_allclose(gp.get_alpha(), post['alpha'], rtol=1e-9, atol=1e-12)
        assert gp.get_hyper_parameters()['mean'].shape == (2, 1 + h_m)          # q1: includes sn
        mo, vo = orc.gp_mean_var(p['X'], hyper, post['alpha'], post['chol'], p['Z'])
        Ny = 2
        mean, cov = gp.predict_batch(p['Z'][:, :Ny], p['Z'][:, Ny:], p['Sigma'])
        np.testing.assert_allclose(mean, mo, rtol=1e-9, atol=1e-12)             # q2: no m(z) added
        gp2 = gp_mpc_b200.GP(p['X'], p['Y'], prior_mean_in_predict=True, **kw)
        mean2, cov2 = gp2.predict_batch(p['Z'][:, :Ny], p['Z'][:, Ny:], p['Sigma'])
        M = np.column_stack([orc.mean_function(hyper[a], p['Z'], func) for a in range(2)])
        np.testing.assert_allclose(mean2, mo + M, rtol=1e-9, atol=1e-12)
        Jfull = orc.gp_mean_jac(p['X'], hyper, post['alpha'], p['Z']) + np.stack([mf.mean_jacobian(hyper[a], p['Z'], func) for a in range(2)], 1)
        np.testing.assert_allclose(cov2, orc.ta_cov(vo, Jfull, p['Sigma']), rtol=1e-8, atol=1e-14)
        A, B = gp2.discrete_linearize(p['Z'][0, :Ny], p['Z'][0, Ny:], None)
        np.testing.assert_allclose(np.hstack([A, B]), Jfull[0], rtol=1e-9, atol=1e-12)
    with pytest.raises(NameError):
        mf.count_mean_params('cubic', 3)
    lbub = mf.mean_bounds(np.array([-1.0, -3.0]), 3, 'linear')                   # inverted reference interval is sorted
    assert (lbub[:, 0] <= lbub[:, 1]).all() and lbub.shape == (4, 2)


@pytest.mark.parametrize('name', ['tank', 'car'])
def test_rollout_device_mapping_equals_the_host_loop(name):
    """GP.rollout hands gpmpc_rollout the standardised start / inputs and the [stdY, meanY, meanX, stdX] map; with an
    engine that restates the C entry in numpy the device path must reproduce the per-step host loop
    (gp_class.py:777-804) to rounding, for both methods, and the default-engine fallback (no `rollout`) is the loop."""
    gp, m = _gp(name, engine_factory=OracleEngineWithRollout)
    d = load_golden('derived', name)
    useq = np.tile(d['u0'], (7, 1)) * (1 + 0.03 * np.arange(7)[:, None])
    rm, rv = gp.rollout(d['x0'], useq, methods=['TA', 'ME'])
    rm_h, rv_h = gp.rollout(d['x0'], useq, methods=['TA', 'ME'], device_rollout=False)
    assert rm.shape == (2, 8, m['Y'].shape[1])
    assert relinf(rm, rm_h) < 1e-12 and relinf(rv, rv_h) < 1e-12
    gp2, _ = _gp(name)                                   # stand-in engine without a rollout entry: host loop
    rm2, rv2 = gp2.rollout(d['x0'], useq, methods=['TA', 'ME'])
    assert np.array_equal(rm2, rm_h) and np.array_equal(rv2, rv_h)


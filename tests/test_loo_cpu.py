"""Leave-one-out cross-validation on CPU: the closed form of oracle/loo_oracle.py against N drop-one refits, its three
gradient forms against each other and against central differences, and the GP class's bookkeeping (units, a prior mean,
validate_loo, the 'objective' option) through an oracle-backed engine."""
import numpy as np
import pytest

import gp_mpc_b200
from gp_mpc_b200.mean_functions import mean_function
from gp_mpc_b200.optimize import bounds_and_init, train_gp_b200
from oracle import gp_oracle as orc
from oracle import loo_oracle as lo
from tests._fake_engine import OracleEngine, problem
from tests._util import load_fixture, projected, relinf


# (mean, var, nlpp) of the closed form against the refits: both carry cond(K) eps (~6e7 tank, ~7e10 car, ~2e6 synthetic)
TOL = {'tank': (1e-10, 1e-9, 1e-10), 'car': (1e-8, 1e-7, 1e-7), 'synthetic': (1e-10, 1e-9, 1e-10)}


@pytest.mark.parametrize('case', ['tank', 'car', 'synthetic'])
def test_closed_form_matches_drop_one_refits(case):
    X, Y, hyper = problem(case)
    tm, tv, tn = TOL[case]
    for a in range(Y.shape[1]):
        cf = lo.closed_form(X, Y[:, a], hyper[a])
        mean, var, nlpp = lo.brute_force(X, Y[:, a], hyper[a])
        assert relinf(cf['mean'], mean) < tm and relinf(cf['var'], var) < tv
        assert abs(cf['nlpp'] - nlpp) <= tn * abs(nlpp)


# (trace form vs eq. 5.13 as an inf-norm and per component, analytic vs five-point differences at the relative step);
# per component because the sn component is up to 3e4 times the others
GRAD = {'tank': (1e-9, 1e-8, 1e-5, 1e-2), 'car': (1e-9, 1e-5, 1e-4, 1e-2), 'synthetic': (1e-12, 1e-9, 1e-7, 1e-3)}


@pytest.mark.parametrize('case', ['tank', 'car', 'synthetic'])
def test_gradient_forms_agree(case):
    X, Y, hyper = problem(case)
    t_tr, t_comp, t_fd, rel = GRAD[case]
    for a in range(min(2, Y.shape[1])):
        theta = hyper[a] * np.linspace(0.9, 1.1, X.shape[1] + 2)
        g = lo.grad_eq513(X, Y[:, a], theta)
        gt = lo.grad_trace(X, Y[:, a], theta)
        assert relinf(gt, g) < t_tr
        assert np.all(np.abs(gt - g) <= t_comp * np.abs(g))
        assert relinf(lo.grad_fd(X, Y[:, a], theta, rel=rel), g) < t_fd


def test_w_matrix_is_symmetric_and_its_trace_gives_the_noise_derivative():
    X, Y, hyper = problem('synthetic')
    W = lo.w_matrix(X, Y[:, 0], hyper[0])
    assert np.array_equal(W, W.T) or relinf(W, W.T) < 1e-14
    sn = hyper[0][-1]
    assert abs(2 * sn * np.trace(W) - lo.grad_eq513(X, Y[:, 0], hyper[0])[-1]) < 1e-9 * abs(2 * sn * np.trace(W))


class LooEngine(OracleEngine):
    """The oracle-backed engine stand-in with gpmpc_loo / gpmpc_loo_nlpp from the closed form; records its calls."""
    created = []

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.calls = []
        LooEngine.created.append(self)

    def nlml(self, a, theta, grad=True):
        self.calls.append('nlml')
        return super().nlml(a, theta, grad)

    def loo(self):
        self.calls.append('loo')
        cfs = [lo.closed_form(self.X, self.Y[:, a], self.hyper[a, :self.Nx + 2]) for a in self.local_outputs]
        return (np.array([c['mean'] for c in cfs]), np.array([c['var'] for c in cfs]),
                np.array([c['nlpp'] for c in cfs]))

    def loo_nlpp(self, a, theta, grad=True):
        self.calls.append('loo_nlpp')
        f = lo.closed_form(self.X, self.Y[:, a], theta)['nlpp']
        return (f, lo.grad_trace(self.X, self.Y[:, a], theta)) if grad else f


def _gp(X, Y, hyper, normalize, meta=None, **kw):
    if meta is not None:
        kw['meta'] = meta
    return gp_mpc_b200.GP(X, Y, gp_method='TA', normalize=normalize, hyper=dict(hyper=hyper),
                          engine_factory=LooEngine, **kw)


@pytest.mark.parametrize('normalize', [True, False])
def test_loo_predict_units(normalize):
    if normalize:                       # the tank fixture is stored standardised, with its meta
        m = load_fixture('tank')
        X, Y, hyper, meta = m['X'], m['Y'], m['hyper'], m['meta']
    else:
        p = orc.synthetic_problem(120, 4, 2, config_id=23)
        X, Y, hyper, meta = p['X'], p['Y'], p['hyper'], None
    gp = _gp(X, Y, hyper, normalize, meta)
    mean, var = gp.loo_predict()
    assert mean.shape == var.shape == Y.shape
    for a in range(Y.shape[1]):
        mu, s2, _ = lo.brute_force(X, Y[:, a], hyper[a])
        if normalize:                   # caller units for the mean, standardised units (q4) for the variance
            mu = mu * meta['stdY'][a] + meta['meanY'][a]
        assert relinf(mean[:, a], mu) < 1e-9 and relinf(var[:, a], s2) < 1e-8


def test_loo_predict_with_a_prior_mean():
    p = orc.synthetic_problem(100, 3, 2, config_id=29)
    X, Y = p['X'], p['Y'] + 2.0
    hyper = np.hstack([p['hyper'], [[1.5], [-0.5]]])            # 'const' prior means
    gp = _gp(X, Y, hyper, False, mean_func='const')
    mean, var = gp.loo_predict()
    for a in range(2):
        m = mean_function(hyper[a], X, 'const')
        mu, s2, _ = lo.brute_force(X, Y[:, a] - m, hyper[a, :5])       # the GP of y - m(X), plus m back
        assert relinf(mean[:, a], mu + m) < 1e-10 and relinf(var[:, a], s2) < 1e-9
        # the residual y - mu = alpha / c does not depend on the prior mean's value
        assert relinf(Y[:, a] - mean[:, a], lo.closed_form(X, Y[:, a] - m, hyper[a, :5])['alpha']
                      / lo.closed_form(X, Y[:, a] - m, hyper[a, :5])['c']) < 1e-10


def test_validate_loo_uses_validates_formulas(capsys):
    m = load_fixture('tank')
    gp = _gp(m['X'], m['Y'], m['hyper'], True, m['meta'])
    smse, mnlp = gp.validate_loo()
    out = capsys.readouterr().out
    assert '# Leave-one-out validation of GP model' in out and '* Num left-out samples: 60' in out
    Ys = m['Y']                         # stored standardised: validate's space
    for a in range(4):
        cf = lo.closed_form(m['X'], Ys[:, a], m['hyper'][a])
        err = Ys[:, a] - cf['mean']
        assert abs(smse[a] - np.mean(err ** 2) / np.std(Ys[:, a])) <= 1e-10 * smse[a]      # q15: over std
        nlp = np.mean(0.5 * np.log(2 * np.pi * cf['var']) + err ** 2 / (2 * cf['var']))
        assert abs(mnlp[a] - nlp) <= 1e-10 * abs(nlp)
        assert abs(mnlp[a] - cf['nlpp'] / 60) <= 1e-10 * abs(nlp)
    # validate with the left-out points as a test set prints the same banner body
    gp.validate(m['X'][:5] * m['meta']['stdZ'] + m['meta']['meanZ'], m['Y'][:5] * m['meta']['stdY'] + m['meta']['meanY'])
    assert '* Num test samples: 5' in capsys.readouterr().out


@pytest.mark.parametrize('opts', [{'objective': 'marginal'}, {'objective': 'loo', 'fit_mean': True},
                                  {'objective': 'loo', 'fit_mean': True, 'jac': 'fd'}])
def test_objective_option_errors_come_before_any_engine_call(opts):
    p = orc.synthetic_problem(40, 3, 2, config_id=3)
    LooEngine.created = []
    with pytest.raises(ValueError):
        gp_mpc_b200.GP(p['X'], p['Y'], mean_func='const', normalize=False, optimizer_opts=opts,
                       engine_factory=LooEngine)
    assert LooEngine.created == []
    eng = LooEngine(40, 3, 2)
    eng.set_data(p['X'], p['Y'])
    with pytest.raises(ValueError):
        train_gp_b200(eng, p['X'], p['Y'], meanFunc='const', optimizer_opts=opts, verbose=False)
    assert eng.calls == []


def test_loo_objective_fit():
    """SLSQP runs on loo_nlpp alone and reaches a stationary point of it (|projected dNLPP/dtheta_j * theta_j| <= 1e-5
    |NLPP|) below the initial point and below the NLML fit on the same objective.  The LOO objective is not convex: on
    other problems a stationary point can lie above the NLML fit's value (DESIGN section 4.13)."""
    p = orc.synthetic_problem(150, 3, 1, config_id=21)
    X, Y = p['X'], p['Y']
    LooEngine.created = []
    gp = gp_mpc_b200.GP(X, Y, normalize=False, optimizer_opts={'objective': 'loo'}, engine_factory=LooEngine)
    fit_eng = LooEngine.created[0]
    assert fit_eng.calls and set(fit_eng.calls) == {'loo_nlpp'}
    ml = gp_mpc_b200.GP(X, Y, normalize=False, engine_factory=LooEngine)
    assert 'loo_nlpp' not in LooEngine.created[-1].calls and 'nlml' in LooEngine.created[-1].calls
    eng = LooEngine(150, 3, 1)
    eng.set_data(X, Y)
    for a in range(1):
        th, th_ml = gp._GP__hyper[a, :5], ml._GP__hyper[a, :5]
        bounds, init = bounds_and_init(X, Y[:, a])
        f, g = eng.loo_nlpp(a, th)
        assert np.abs(projected(g, th, bounds) * th).max() < 1e-5 * abs(f)
        assert f < eng.loo_nlpp(a, init, grad=False) and f < eng.loo_nlpp(a, th_ml, grad=False)

"""oracle/rollout_oracle_ld.py, the long-double restatement of the device roll-outs, against the float64 oracles it must
agree with (rollout_grad_oracle, sample_oracle) on one LAPACK factor, against central differences of itself, and its
sums of |terms| against its values."""
import numpy as np
import pytest
from scipy.linalg import solve_triangular

from oracle import gp_oracle as orc
from oracle import rollout_oracle
from oracle import sample_oracle as so
from oracle.rollout_grad_oracle import rollout_grad
from oracle.rollout_oracle_ld import LD, MARGIN, rollout_ld, sample_ld
from tests._util import load_fixture, load_golden, relinf

# rollout_ld against the float64 oracles on the same factor, normalised by rollout_ld's sums of |terms|: the float64
# oracles round on that scale too (tank's means cancel 1e5-fold, car's more), so a plain relative error would measure them
BAR = 1e-12
# rollout_ld's tangents against its own central differences at a step of 1e-5: tank's means cancel 1e5-fold, so the
# quotient carries ~1e-19 x 1e5 / 1e-5 of rounding besides the O(1e-10) truncation
FD_BAR = 1e-7


def _problem(name):
    """Model dict (X, Y, hyper, alpha, chol, normalize, meta) with LAPACK's factor, its L^-1, and a start x0, inputs
    u0 (caller units) and x_ref."""
    if name == 'nx17':
        p = orc.synthetic_problem(150, 17, 9, config_id=17)
        m = dict(X=p['X'], Y=p['Y'], hyper=p['hyper'], normalize=False)
        x0, u0 = 0.5 * p['Z'][0, :9], 0.5 * p['Z'][0, 9:]
    else:
        m = load_fixture(name)
        d = load_golden('derived', name)
        x0, u0 = np.asarray(d['x0'], dtype=np.float64), np.asarray(d['u0'], dtype=np.float64)
    post = orc.postfit(m['X'], m['Y'], m['hyper'], lapack_general_solve=False)
    N = m['X'].shape[0]
    linv = np.stack([solve_triangular(c, np.eye(N), lower=True) for c in post['chol']])
    model = dict(X=m['X'], Y=m['Y'], hyper=m['hyper'], alpha=post['alpha'], chol=post['chol'],
                 normalize=m['normalize'], meta=m.get('meta'))
    return model, linv, x0, u0, 0.9 * x0 + 0.1


def _units(model):
    Ny, Nx = model['hyper'].shape[0], model['X'].shape[1]
    Nu = Nx - Ny
    if model['normalize']:
        st = model['meta']
        return tuple(np.asarray(st[k], dtype=np.float64) for k in ('meanX', 'stdX', 'meanU', 'stdU', 'meanY', 'stdY'))
    return np.zeros(Ny), np.ones(Ny), np.zeros(Nu), np.ones(Nu), np.zeros(Ny), np.ones(Ny)


def _engine_args(model, x0, U, K=None, x_ref=None):
    """What GP.rollout hands the engine for one trajectory: z0 (1, Nx), U (1, Nt, Nu), Sigma0, scale, uscale."""
    mX, sX, mU, sU, mY, sY = _units(model)
    Ny, Nx = model['hyper'].shape[0], model['X'].shape[1]
    u0 = U[0] if K is None else K @ (x0 - x_ref)
    z0 = np.concatenate([(x0 - mX) / sX, (u0 - mU) / sU])[None]
    S = np.eye(Nx) * 1e-6
    S[:Ny, :Ny] = np.diag(model['hyper'][:, Nx + 1] ** 2)
    scale = np.stack([sY, mY, mX, sX]) if model['normalize'] else None
    uscale = np.stack([mU, sU]) if (model['normalize'] and K is not None) else None
    return z0, ((U - mU) / sU)[None], S[None], scale, uscale


def _to_caller(o, model, x0, K, x_ref, absolute=False):
    """rollout_ld's engine-unit outputs (one trajectory) as rollout_grad_oracle's caller-unit dict (rows 1..Nt);
    ``absolute``: the same map of the sums of |terms| (o's 's_' entries, |coefficients|)."""
    mX, sX, mU, sU, mY, sY = _units(model)
    Ny, Nx = model['hyper'].shape[0], model['X'].shape[1]
    Nu = Nx - Ny
    g = (lambda k: np.asarray(o['s_' + k][0], dtype=np.float64)) if absolute else \
        (lambda k: np.asarray(o[k][0], dtype=np.float64))
    if absolute:
        sX, sU, sY, mY = np.abs(sX), np.abs(sU), np.abs(sY), np.abs(mY)
        K = None if K is None else np.abs(K)
    res = dict(mean=g('mean') * sY + mY, var=g('var') * sY ** 2)
    for k, f in (('mean', sY), ('var', sY ** 2)):
        D = g('d' + k)                                                     # (Nt, Ny, P)
        Du0 = D[..., Ny:Nx] / sU                                           # d / d u0 (caller)
        dx0 = D[..., :Ny] / sX
        if K is None:
            res['d%s_dx0' % k] = dx0 * f[:, None]
            rest = D[..., Nx:].reshape(D.shape[0], Ny, -1, Nu) / sU
            res['d%s_du' % k] = np.concatenate([Du0[:, :, None], rest], 2) * f[:, None, None]
        else:
            xt = np.abs(x0 - x_ref) if absolute else x0 - x_ref
            res['d%s_dx0' % k] = (dx0 + Du0 @ K) * f[:, None]
            dK = D[..., Nx:].reshape(D.shape[0], Ny, Nu, Ny) + Du0[..., None] * xt[None, None, None, :]
            res['d%s_dK' % k] = dK * f[:, None, None]
    return res


@pytest.mark.parametrize('fb', [False, True])
@pytest.mark.parametrize('meth', ['TA', 'ME'])
@pytest.mark.parametrize('name', ['tank', 'car', 'nx17'])
def test_rollout_ld_equals_the_float64_oracle(name, meth, fb):
    """Means, variances and every tangent against rollout_grad_oracle (caller units) on one LAPACK factor, open loop and
    with a fixed feedback gain."""
    model, linv, x0, u0, x_ref = _problem(name)
    Ny, Nx = model['hyper'].shape[0], model['X'].shape[1]
    Nu, Nt = Nx - Ny, 5
    U = np.tile(u0, (Nt, 1)) * (1 + 0.03 * np.arange(Nt)[:, None])
    K = None
    if fb:
        A, Bm = orc.discrete_linearize(model, x0, U[0])
        K = rollout_oracle.lqr_gain(A, Bm, np.eye(Ny), np.eye(Nu))[0]
    z0, Ue, S0, scale, uscale = _engine_args(model, x0, U, K, x_ref)
    o = rollout_ld(model['X'], model['hyper'], model['alpha'], linv, z0, Ue, S0, meth, scale, K,
                   x_ref if fb else None, uscale, tangents=True)
    got = _to_caller(o, model, x0, K, x_ref)
    scale = _to_caller(o, model, x0, K, x_ref, absolute=True)
    ref = rollout_grad(model, x0, U, meth, feedback=fb, x_ref=x_ref, K=K)
    for k, v in got.items():
        d = np.abs(v - ref[k][1:])
        assert not np.any(d[scale[k] == 0]), k                          # structural zeros (later inputs) on both sides
        err = np.max(np.divide(d, scale[k], out=np.zeros_like(d), where=scale[k] > 0))
        assert err <= BAR, (k, err)


def _central(f, x, rel=1e-5):
    """Central differences of f (an array of np.longdouble) at x in every coordinate of x."""
    cols = []
    for p in range(x.size):
        h = LD(rel) * max(LD(1), abs(x.flat[p]))
        xp, xm = x.copy(), x.copy()
        xp.flat[p] += h
        xm.flat[p] -= h
        cols.append((f(xp) - f(xm)) / (2 * h))
    return np.stack(cols, -1)


@pytest.mark.parametrize('fb', [False, True])
@pytest.mark.parametrize('meth', ['TA', 'ME'])
def test_tangents_equal_long_double_central_differences(meth, fb):
    """dmean, dvar against central differences of rollout_ld itself in every parameter (z0, U rows 1.. or the entries of
    K), on the normalised tank model with x_ref and uscale."""
    model, linv, x0, u0, x_ref = _problem('tank')
    Ny, Nx = model['hyper'].shape[0], model['X'].shape[1]
    Nu, Nt = Nx - Ny, 4
    U = np.tile(u0, (Nt, 1)) * (1 + 0.03 * np.arange(Nt)[:, None])
    K = 0.2 * np.random.default_rng(5).standard_normal((Nu, Ny)) if fb else None
    z0, Ue, S0, scale, uscale = _engine_args(model, x0, U, K, x_ref)
    args = (model['X'], model['hyper'], model['alpha'], np.asarray(linv, dtype=LD))
    xr = x_ref if fb else None
    o = rollout_ld(*args, z0, Ue, S0, meth, scale, K, xr, uscale, tangents=True)
    if fb:
        theta = np.concatenate([z0[0], K.ravel()]).astype(LD)
        split = lambda th: (th[None, :Nx], Ue, th[Nx:].reshape(Nu, Ny))
    else:
        theta = np.concatenate([z0[0], Ue[0, 1:].ravel()]).astype(LD)
        split = lambda th: (th[None, :Nx], np.concatenate([Ue[:, :1], th[Nx:].reshape(1, Nt - 1, Nu)], 1), None)

    def f(th):
        z, Uh, Kh = split(th)
        r = rollout_ld(*args, z, Uh, S0, meth, scale, K if Kh is None else Kh, xr, uscale)
        return np.concatenate([r['mean'][0].ravel(), r['var'][0].ravel()])

    fd = _central(f, theta)
    an = np.concatenate([o['dmean'][0].reshape(Nt * Ny, -1), o['dvar'][0].reshape(Nt * Ny, -1)])
    err = relinf(np.asarray(an, dtype=np.float64), np.asarray(fd, dtype=np.float64))
    assert err <= FD_BAR, err


@pytest.mark.parametrize('fb', [False, True])
@pytest.mark.parametrize('name', ['tank', 'car'])
def test_sample_ld_equals_the_sample_oracle(name, fb):
    """Samples and kept flags of sample_ld along the oracle's own inputs equal sample_oracle.rollout_sample's (with xi,
    scale, and with feedback x_ref and uscale)."""
    model, linv, x0, u0, x_ref = _problem(name)
    Ny, Nx = model['hyper'].shape[0], model['X'].shape[1]
    Nu, Nt, B = Nx - Ny, 12, 3
    rng = np.random.default_rng(4)
    U = np.tile(u0, (Nt, 1)) * (1 + 0.03 * np.arange(Nt)[:, None])
    K = 0.1 * rng.standard_normal((Nu, Ny)) if fb else None
    z0, Ue, _, scale, uscale = _engine_args(model, x0, U, K, x_ref)
    z0 = z0 + 0.02 * rng.standard_normal((B, Nx))
    Ue = np.repeat(Ue, B, 0)
    eps, xi = rng.standard_normal((B, Nt, Ny)), rng.standard_normal((B, Nt, Ny))
    sm, z_out, kept = so.rollout_sample(model, linv, z0, Ue, eps, xi, scale, K, x_ref if fb else None, uscale)
    o = sample_ld(model['X'], model['hyper'], model['alpha'], linv, z_out, eps, xi, kept=kept)
    sure = o['margin'] >= MARGIN                 # tank's slow dynamics revisit nearly the same inputs: d ~ DELTA sf2
    assert sure[:, 0].all()
    assert np.array_equal(o['kept'][sure], kept[sure].astype(bool))
    err = np.abs(np.asarray(o['samples'] - sm, dtype=np.float64)) / np.asarray(o['s_samples'], dtype=np.float64)
    assert err.max() <= BAR, err.max()


def test_sums_of_terms_bound_their_values():
    """Every s_ value is >= |value| (open loop and feedback, TA and ME, with tangents), and every sample's sum bounds it."""
    model, linv, x0, u0, x_ref = _problem('tank')
    Ny, Nx = model['hyper'].shape[0], model['X'].shape[1]
    Nu, Nt = Nx - Ny, 4
    U = np.tile(u0, (Nt, 1))
    K = 0.2 * np.random.default_rng(5).standard_normal((Nu, Ny))
    args = (model['X'], model['hyper'], model['alpha'], np.asarray(linv, dtype=LD))
    for Kf in (None, K):
        z0, Ue, S0, scale, uscale = _engine_args(model, x0, U, Kf, x_ref)
        for meth in ('TA', 'ME'):
            o = rollout_ld(*args, z0, Ue, S0, meth, scale, Kf, x_ref if Kf is not None else None, uscale, tangents=True)
            for k in ('mean', 'var', 'cov_last', 'dmean', 'dvar'):
                assert np.all(o['s_' + k] >= np.abs(o[k])), (meth, Kf is None, k)
    rng = np.random.default_rng(1)
    z0, Ue, _, scale, _ = _engine_args(model, x0, np.tile(u0, (8, 1)))
    eps = rng.standard_normal((1, 8, Ny))
    _, z_out, _ = so.rollout_sample(model, linv, z0, Ue, eps, None, scale)
    o = sample_ld(model['X'], model['hyper'], model['alpha'], linv, z_out, eps)
    assert np.all(o['s_samples'] >= np.abs(o['samples']))

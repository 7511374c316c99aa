"""Shared helpers for the test-suite: fixture loading, error norms, finite differences, shared bars and test data.
Imports nothing beyond numpy at module level (smoke(), tools/ and oracle/make_golden_*.py import it)."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def unpack_lower(packed, n, symmetric=False):
    packed = np.asarray(packed)
    out = np.zeros(packed.shape[:-1] + (n, n))
    i, j = np.tril_indices(n)          # row-major lower order (index work: bit-exact)
    out[..., i, j] = packed
    if symmetric:
        out[..., j, i] = packed
    return out


def load_fixture(name):
    """The reference's saved model gp_<name>_example.json as a model dict."""
    z = np.load(os.path.join(GOLDEN, 'fixture_%s.npz' % name))
    N = z['X'].shape[0]
    m = dict(X=z['X'], Y=z['Y'], hyper=z['hyper'], alpha=z['alpha'],
             chol=unpack_lower(z['chol_packed'], N),
             invK=unpack_lower(z['invK_packed'], N, symmetric=True),
             length_scale=z['length_scale'], signal_var=z['signal_var'],
             noise_var=z['noise_var'], mean=z['mean'],
             normalize=bool(z['normalize']), mean_func='zero')
    if 'invK_full' in z.files:
        m['invK'] = z['invK_full']
    if m['normalize']:
        m['meta'] = {k[5:]: z[k] for k in z.files if k.startswith('meta_')}
        for k in ('xlb', 'xub', 'ulb', 'uub'):
            m[k] = z[k]
    return m


def load_golden(kind, name):
    return np.load(os.path.join(GOLDEN, '%s_%s.npz' % (kind, name)))


def relinf(a, b):
    """batch-infinity-norm relative error  max|a-b| / max|b|  (SURVEY 8d gate)."""
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    den = np.abs(b).max()
    return np.abs(a - b).max() / (den if den > 0 else 1.0)


# bars on the largest error of the prediction and its input derivatives normalised by the sum of |terms|, per output
# family (measured maxima in the docstring of test_predict_derivs_shapes_gpu)
PREDICT_TOL = dict(mean=1e-15, var=1e-16, cov=1e-16, jac=1e-15, dvar_dz=1e-16, dcov_dz=1e-16, hess=1e-14,
                   d2var_dz2=1e-16, d3mean_dz3=1e-14, d2cov_dz2=1e-16)
# bar on the predict product's variance against long double over its sum of |terms|: a stale band is an O(1) error; the
# fp64 product measured at most 2.7e-19 of the scale
PREDICT_VAR_TOL = 1e-16


def normalised(x, ref, scale):
    """Largest |x - ref| / scale over the entries, in long double; entries whose sum of |terms| is 0 must be exactly 0 on
    both sides."""
    d = np.abs(np.asarray(x, dtype=np.longdouble) - np.asarray(ref, dtype=np.longdouble))
    assert not np.any(d[scale == 0]), 'a nonzero entry where the sum of |terms| is 0'
    return float(np.max(np.divide(d, scale, out=np.zeros_like(d), where=scale > 0), initial=0.0))


def central(f, p, rel):
    """Central differences of f (returning mean, var) at the parameter array p, one entry at a time."""
    p = np.asarray(p, dtype=np.float64)
    dm, dv = [], []
    for j in np.ndindex(p.shape):
        h = rel * max(1.0, abs(p[j]))
        pp = p.copy(); pp[j] += h
        pm = p.copy(); pm[j] -= h
        (mp, vp), (mm, vm) = f(pp), f(pm)
        dm.append((mp - mm) / (2 * h)); dv.append((vp - vm) / (2 * h))
    sh = p.shape
    return (np.moveaxis(np.array(dm), 0, -1).reshape(dm[0].shape + sh),
            np.moveaxis(np.array(dv), 0, -1).reshape(dv[0].shape + sh))


def d4(fun, h):
    """Fourth-order central differences of fun (returning a dict of arrays) at step h."""
    r = {k: fun(k * h) for k in (-2, -1, 1, 2)}
    return {key: (r[-2][key] - 8 * r[-1][key] + 8 * r[1][key] - r[2][key]) / (12 * h) for key in r[1]}


def projected(g, th, bounds):
    """The gradient with the components that point out of an active bound zeroed (active: within 1e-8 of its range)."""
    tol = 1e-8 * (bounds[:, 1] - bounds[:, 0])
    return np.where((th <= bounds[:, 0] + tol) & (g > 0), 0.0, np.where((th >= bounds[:, 1] - tol) & (g < 0), 0.0, g))


def assert_same(a, b):
    """The arrays of two sequences are equal bit for bit, pair by pair."""
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def free_port():
    import socket
    s = socket.socket(); s.bind(('127.0.0.1', 0)); p = s.getsockname()[1]; s.close(); return p


def trajectories(name, nb, Nt, cyclic):
    """nb starts around the fixture's stored x0 and Nt inputs each around its u0 (caller units), and x_ref = 0.9 x0 + 0.1.
    Trajectory b scales x0 by 1 + 0.05 b and its inputs by 1 + 0.02 b, or with cyclic by 1 + 0.01 (b mod 23)
    - 0.004 (b mod 7) and 1 + 0.005 (b mod 11); step t's inputs are further scaled by 1 + 0.03 t."""
    d = load_golden('derived', name)
    x0 = np.asarray(d['x0'], dtype=np.float64)
    u0 = np.asarray(d['u0'], dtype=np.float64)
    if cyclic:
        X0 = np.stack([x0 * (1 + 0.01 * (b % 23) - 0.004 * (b % 7)) for b in range(nb)])
        U = np.stack([np.tile(u0, (Nt, 1)) * (1 + 0.03 * np.arange(Nt)[:, None] + 0.005 * (b % 11)) for b in range(nb)])
    else:
        X0 = np.stack([x0 * (1 + 0.05 * b) for b in range(nb)])
        U = np.stack([np.tile(u0, (Nt, 1)) * (1 + 0.03 * np.arange(Nt)[:, None] + 0.02 * b) for b in range(nb)])
    return X0, U, 0.9 * x0 + 0.1

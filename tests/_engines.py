"""Helpers that drive the real engine: fitted handles and GPs, and the kernel-selection rules of gpmpc.cu that the
shape tests restate to know which instantiation a case reaches.  Importing this module needs neither the built library
nor a GPU; creating an Engine needs both."""
import numpy as np
import pytest

import gp_mpc_b200
from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._util import load_fixture


def built_lib():
    """The library binding after build(): compiles libgpmpc.so if it is missing or stale."""
    import __graft_entry__ as g
    g.build()
    return L


def fit(X, Y, hyper, with_info=False, **kw):
    """An engine on device 0 holding X, Y and hyper, factorised; with_info also returns factorize's per-output info.
    kw go to Engine (capacity, ...)."""
    eng = L.Engine(X.shape[0], X.shape[1], Y.shape[1], device=0, **kw)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)
    info = eng.factorize()
    return (eng, info) if with_info else eng


def problem(case):
    """X, Y, hyper of a stored fixture ('tank', 'car'), or of the synthetic problem of case = (N, Nx, Ny)."""
    if case in ('tank', 'car'):
        m = load_fixture(case)
        return m['X'], m['Y'], m['hyper']
    N, Nx, Ny = case
    p = orc.synthetic_problem(N, Nx, Ny, config_id=N + Nx)
    return p['X'], p['Y'], p['hyper']


def synthetic_engine(N, Nx, Ny, seed, H):
    """A factorised engine on orc.synthetic_problem(N, Nx, Ny, config_id=seed, H=H), and the problem."""
    p = orc.synthetic_problem(N, Nx, Ny, config_id=seed, H=H)
    eng, info = fit(p['X'], p['Y'], p['hyper'], with_info=True)
    assert not info.any()
    return eng, p


def sample_engine(name):
    """(engine, model dict) for a fixture or the synthetic problem of the sampled roll-out tests."""
    if name == 'synthetic':                              # N = 1000, Nx = 8, Ny = 6 (Nu = 2)
        p = orc.synthetic_problem(1000, 8, 6, config_id=4)
        m = dict(X=p['X'], Y=p['Y'], hyper=p['hyper'], normalize=False)
    else:
        m = load_fixture(name)
    return fit(m['X'], m['Y'], m['hyper']), m


def gp_from_fixture(name):
    """A GP on the device built from a stored fixture with its stored factor, and the fixture."""
    m = load_fixture(name)
    kw = dict(mean_func='zero', gp_method='TA', normalize=m['normalize'],
              hyper=dict(hyper=m['hyper'], invK=m['invK'], alpha=m['alpha'], chol=m['chol'],
                         length_scale=m['length_scale'], signal_var=m['signal_var'],
                         noise_var=m['noise_var'], mean=m['mean']))
    if m['normalize']:
        kw.update(meta=m['meta'], xlb=m['xlb'], xub=m['xub'], ulb=m['ulb'], uub=m['uub'])
    return gp_mpc_b200.GP(m['X'], m['Y'], **kw), m


def lqr_gain(gp, X0, U):
    """The GP's LQR gain at the first start and input, with identity weights."""
    Ny, Nu = X0.shape[1], U.shape[2]
    return gp._GP__lqr_gains(X0[:1], U[:1, 0], np.eye(Ny), np.eye(Nu))[0]


def ccs(ptr):
    """(nrow, ncol, colind, rows) of a CasADi compressed-column sparsity pattern."""
    nrow, ncol = ptr[0], ptr[1]
    colind = [ptr[2 + k] for k in range(ncol + 1)]
    rows = [ptr[2 + ncol + 1 + k] for k in range(colind[-1])]
    return nrow, ncol, colind, rows


# ------------------------------------------------------------------ shape selection
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def require(ok, what):
    if not ok:
        pytest.skip('this device (%d SMs) does not put the case on %s' % (sms(), what))


def npad(n):
    return -(-n // 128) * 128


def ks_chunk(npad, nloc, nx):
    """gpmpc.cu:807-811."""
    if npad < 8192:
        return 128
    return 1024 if (nloc >= 2 and nx <= 12) else 512


def gemm_feed(mt, nt, lower, bt, batch, sms, small_tiles=None):
    """gemm128's choice (gpmpc.cu:206-218) for a product of mt x nt 128x128 tiles: '64x32', 'tma' or '128x64'.
    The tile count is in 128x64 tiles and includes the batch; small_tiles defaults to 4 * SMs (gpmpc.cu:417)."""
    tiles = batch * (mt * (mt + 1) if lower else 2 * mt * nt)
    if tiles < (4 * sms if small_tiles is None else small_tiles):
        return '64x32', tiles
    if bt and tiles >= 4 * sms:
        return 'tma', tiles
    return '128x64', tiles

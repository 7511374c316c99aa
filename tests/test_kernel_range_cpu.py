"""The kernel evaluation of the K build and the ks kernel restated on the CPU (tests/_kernel_range.py), no GPU:

A1. exp2_t2lvl (kernels.cuh) operation for operation, with fma done exactly, against mpmath at 120 bits over its
    documented domain -1020 <= t <= 1000: both tables correctly rounded, every result within EXP2_ULP ulp, and the
    clamp's argument -1020 giving 2^-1020 exactly.
A2. The rounding-error bounds on t that the GPU tests (test_kernel_range_gpu.py) hold each kernel to, checked against
    numpy emulations of each kernel's formula, including a K build centred on a stale mean."""
import math

import numpy as np
import pytest

from tests import _kernel_range as kr

mpmath = pytest.importorskip('mpmath')


def _exact_exp2(t):
    with mpmath.workprec(120):
        return mpmath.power(2, mpmath.mpf(t))


def _ulps(v, t):
    ex = _exact_exp2(t)
    with mpmath.workprec(120):
        return float(abs(mpmath.mpf(v) - ex) / kr.ulp(float(ex)))


def test_exp2_tables_are_correctly_rounded():
    for k in range(16):
        for tab, den in ((kr.T1, 16), (kr.T2, 256)):
            with mpmath.workprec(120):
                ex = mpmath.power(2, mpmath.mpf(k) / den)
                assert abs(mpmath.mpf(tab[k]) - ex) <= mpmath.mpf(kr.ulp(tab[k])) / 2, (den, k)


def _arguments():
    """Random arguments over the domain, and around the rounding boundaries of n = rint(256 t): the table indices
    repeat with period 1 in t, so all 256 residues of n at a few integer parts reach every table pair, each at the
    boundary k/256 itself, at the halfway points k/256 +- 1/512 (where rint ties to even), and 1e-13 either side."""
    rng = np.random.default_rng(5)
    ts = list(rng.uniform(-1020.0, 1000.0, 2000)) + list(rng.uniform(-2.0, 2.0, 500))
    for e in (-1019, -513, -1, 0, 37, 998):
        for k in range(256):
            b = e + k / 256.0
            for off in (0.0, 1 / 512, -1 / 512, 1e-13, -1e-13, 1 / 512 + 1e-13, 1 / 512 - 1e-13, -1 / 512 + 1e-13):
                t = b + off
                if -1020.0 <= t <= 1000.0:
                    ts.append(t)
    ts += [-1020.0, -1020.0 + 1 / 512 - 1e-12, 0.0, -0.0, 1000.0, 999.998]
    return ts


def test_exp2_t2lvl_error_over_its_domain():
    """Measured: 2.75 ulp at most over these arguments (the figure quoted in kernels.cuh and DESIGN.md)."""
    worst = 0.0
    for t in _arguments():
        worst = max(worst, _ulps(kr.exp2_t2lvl(t), t))
    assert worst <= kr.EXP2_ULP, worst
    assert worst > 2.0, worst                       # the figure quoted in the docs is a measured maximum, not slack


def test_exp2_t2lvl_ends_of_its_domain():
    assert kr.exp2_t2lvl(-1020.0) == kr.K_MIN == 2.0 ** -1020     # the clamp's documented result, bit for bit
    assert kr.exp2_t2lvl(0.0) == 1.0 and kr.exp2_t2lvl(-0.0) == 1.0
    for t in (-1019.5, -1000.25, 512.0, 1000.0):
        assert _ulps(kr.exp2_t2lvl(t), t) <= kr.EXP2_ULP, t
    assert kr.exp2_t2lvl(-40.0) == 2.0 ** -40 and kr.exp2_t2lvl(17.0) == 2.0 ** 17


def _t_mp(xi, xj, ell, sf2):
    with mpmath.workprec(160):
        s = mpmath.mpf(0)
        for a, b, l in zip(xi, xj, ell):
            s += ((mpmath.mpf(a) - mpmath.mpf(b)) / mpmath.mpf(l)) ** 2
        return mpmath.log(mpmath.mpf(sf2), 2) - s / (2 * mpmath.log(2))


def _designs():
    rng = np.random.default_rng(11)
    out = []
    for Nx, ell, sf2, shift, stale in ((1, 0.01, 1.0, 0.0, 0.0), (4, 1.0, 2.0 ** -40, 0.0, 0.0),
                                       (8, 0.3, (2 ** 6 * 3.0) ** 2, 5.0, 0.0), (17, 3.0, 1.0, 0.0, 0.0),
                                       (4, 1.0, 1.0, 1000.0, 1000.0),          # centre left at the old mean
                                       (32, 0.05, 1.0, 0.0, 0.0)):
        X = rng.standard_normal((24, Nx)) + shift
        ellv = ell * rng.uniform(0.5, 2.0, Nx)
        mu = X.mean(0) - stale
        out.append((X, ellv, sf2, mu))
    return out


@pytest.mark.parametrize('case', range(6))
def test_kbuild_t_bound_holds_on_an_emulation(case):
    """The K build's expansion t = (q_i + q_j) + u_i . u_j emulated in numpy (separate multiply and add, not fma: more
    roundings than the kernel) against t at 160 bits: every pair within kbuild_bound, and the bound not loose by more
    than a few hundred times where cancellation is large (the stale-centre design)."""
    X, ell, sf2, mu = _designs()[case]
    t, bnd, Ui, _ = kr.kbuild_t(X, X, mu, ell, sf2)
    worst = 0.0
    for i in range(X.shape[0]):
        for j in range(X.shape[0]):
            err = abs(t[i, j] - float(_t_mp(X[i], X[j], ell, sf2)))
            assert err <= bnd[i, j], (i, j, err, bnd[i, j])
            worst = max(worst, err / bnd[i, j])
    if case == 4:
        assert np.max(np.einsum('nd,nd->n', Ui, Ui)) > 1e6       # |u|^2 from the stale centre: digits lost
        assert worst > 1e-3, worst


@pytest.mark.parametrize('case', range(6))
def test_ks_t_bound_holds_on_an_emulation(case):
    """The ks kernel's direct differences of scaled coordinates, emulated in numpy, against t at 160 bits."""
    X, ell, sf2, _ = _designs()[case]
    Z = X[::3] + 0.1 * np.random.default_rng(case).standard_normal(X[::3].shape)
    te, bnd = kr.ks_t(X, Z, ell, sf2)
    for i in range(X.shape[0]):
        for h in range(Z.shape[0]):
            err = abs(te[i, h] - float(_t_mp(X[i], Z[h], ell, sf2)))
            assert err <= bnd[i, h], (i, h, err, bnd[i, h])


def test_long_double_reference_of_t():
    """t_exact, the GPU tests' reference, agrees with 160-bit t to far inside the kernels' bounds."""
    if not kr.LD_OK:
        pytest.skip('long double has no 64-bit significand here')
    X, ell, sf2, mu = _designs()[2]
    sf = math.sqrt(sf2)
    te = kr.t_exact(X, X, ell, sf)
    _, bnd, _, _ = kr.kbuild_t(X, X, mu, ell, sf2)
    for i in range(0, X.shape[0], 3):
        for j in range(X.shape[0]):
            with mpmath.workprec(160):
                num, den = te[i, j].as_integer_ratio()
                err = abs(mpmath.mpf(num) / den - _t_mp(X[i], X[j], ell, sf * sf))
            assert float(err) <= 1e-2 * bnd[i, j]


def test_entry_bound_below_and_at_the_clamp():
    """rel_bound turns |dt| into a relative entry error; an exact t below -1020 - bound clamps to 2^-1020."""
    assert kr.rel_bound(0.0) == kr.EXP2_ULP * kr.EPS
    assert kr.rel_bound(1e-12) == pytest.approx(kr.EXP2_ULP * kr.EPS + math.log(2) * 1e-12, rel=1e-6)
    X = np.array([[0.0], [1.0], [40.0]])
    t, bnd, _, _ = kr.kbuild_t(X, X, X.mean(0), np.array([0.01]), 1.0)
    assert t[0, 2] < kr.T_MIN - bnd[0, 2] and t[0, 1] < kr.T_MIN - bnd[0, 1]

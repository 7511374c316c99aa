"""The kernel evaluation sf2 exp(-1/2 |(x - z)/ell|^2) = 2^t of the K build and the ks kernel, restated on the CPU:
the two-level-table exp2 bit for bit (exp2_t2lvl, kernels.cuh) and a rounding-error bound on t for each kernel's own
operation order.  The CPU tests check both against mpmath; the GPU tests hold every device entry to the same bounds.

Bounds (eps = 2^-52, u_r = eps / 2), in the variables the kernels use:

* K build (kbuild_dmma_kernel): u_i = sqrt(log2 e) (x_i - mu) / ell, q_i = -1/2 |u_i|^2 + 1/2 log2 sf2 and
  t = (q_i + q_j) + u_i . u_j.  Each u_id carries 4 roundings (the constant, 1/ell, x - mu, the product), the fma chain
  of |u|^2 and the DMMA dot product at most Nx each, and q and the two adds one each, so with gamma = (Nx + 6) eps
      |t - t*| <= gamma (|u_i|^2 + |u_j|^2 + sum_d |u_id u_jd| + |log2 sf2|) + 4 eps.
  The bound grows with |u|^2 measured from the centre mu: the expansion cancels, direct differences do not.
* ks kernel (ks_tile_kernel): xs = x * (1/ell), zs = z * (1/ell), df = xs - zs, dist = sum df^2 (two fma chains),
  te = fma(-log2(e)/2, dist, log2 sf2).  The differences of the scaled coordinates carry an absolute error of
  u_r (|xs| + |zs|) + u_r |df| each, so
      |te - t*| <= log2(e)/2 (2 sum_d |df_d| (2 u_r (|xs_d| + |zs_d|) + 2 u_r |df_d|) + (Nx/2 + 3) eps dist)
                   + eps |te| + 4 eps   (eps |te|: the rounded argument and the device log2 of sf).
  It grows with |t| eps: the argument itself is rounded.

The entry 2^t is then within EXP2_ULP ulp of 2^t~ (exp2_t2lvl), so its relative error against the exact kernel value
is at most EXP2_ULP eps + expm1(ln 2 |t - t*|).  Below t = -1020 both kernels clamp: the entry is 2^-1020 exactly."""
import math
import struct
from fractions import Fraction

import numpy as np

EPS = 2.0 ** -52
SQRT_LOG2E = 1.2011224087864498          # the K build's constant (kernels.cuh)
HALF_LOG2E = 0.72134752044448170         # the ks kernel's constant
T_MIN = -1020.0                          # the lower clamp of both kernels
K_MIN = 2.0 ** -1020                     # 2^T_MIN, the clamp's result
EXP2_ULP = 3.0                           # exp2_t2lvl's error bound in ulp (measured max in test_kernel_range_cpu)

# 2^(k/16) and 2^(m/256), k, m = 0..15: the two tables of exp2_t2lvl (c_exp2_tab, c_exp2_tab2)
T1 = (1.0, 1.0442737824274138, 1.0905077326652577, 1.1387886347566916, 1.189207115002721,
      1.241857812073484, 1.2968395546510096, 1.3542555469368927, 1.4142135623730951,
      1.4768261459394993, 1.5422108254079407, 1.6104903319492543, 1.681792830507429,
      1.7562521603732995, 1.8340080864093424, 1.9152065613971474)
T2 = (1, 1.0027112750502025, 1.0054299011128027, 1.0081558981184175, 1.0108892860517005, 1.0136300849514894,
      1.0163783149109531, 1.0191339960777379, 1.0218971486541166, 1.0246677928971357, 1.0274459491187637,
      1.030231637686041, 1.0330248790212284, 1.0358256936019572, 1.0386341019613787, 1.0414501246883161)
POLY = (0.009618129107628477, 0.05550410866482158, 0.24022650695910072, 0.6931471805599453, 1.0)


def fma(a, b, c):
    """a * b + c with one rounding."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _words(x):
    lo, hi = struct.unpack('<iI', struct.pack('<d', x))
    return hi, lo


def exp2_t2lvl(t):
    """exp2_t2lvl (kernels.cuh) operation for operation: the result the device computes for the double t."""
    SH = 6755399441055744.0
    s = fma(t, 256.0, SH)
    n = _words(s)[1]                                  # __double2loint: signed low word
    f = fma(s - SH, -0.00390625, t)
    p = POLY[0]
    for c in POLY[1:]:
        p = fma(p, f, c)
    p *= T1[(n >> 4) & 15]
    p *= T2[n & 15]
    hi, lo = _words(p)
    hi = (hi + ((n >> 8) << 20)) & 0xFFFFFFFF
    return struct.unpack('<d', struct.pack('<iI', lo, hi))[0]


def ulp(x):
    """The spacing of doubles at |x| (normal range)."""
    return 2.0 ** (math.frexp(abs(x))[1] - 53)


def kbuild_t(Xi, Xj, mu, ell, sf2):
    """The K build's t (numpy order, no fma) and its bound, for all pairs of rows of Xi and Xj: (t, bound, u_i, u_j)."""
    sc = SQRT_LOG2E / ell
    Ui = (Xi - mu) * sc
    Uj = (Xj - mu) * sc
    l2 = math.log2(sf2)
    qi = -0.5 * np.einsum('nd,nd->n', Ui, Ui) + 0.5 * l2
    qj = -0.5 * np.einsum('nd,nd->n', Uj, Uj) + 0.5 * l2
    t = (qi[:, None] + qj[None, :]) + Ui @ Uj.T
    return t, kbuild_bound(Ui, Uj, sf2), Ui, Uj


def kbuild_bound(Ui, Uj, sf2):
    Nx = Ui.shape[1]
    g = (Nx + 6) * EPS
    ni = np.einsum('nd,nd->n', Ui, Ui)
    nj = np.einsum('nd,nd->n', Uj, Uj)
    return g * (ni[:, None] + nj[None, :] + np.abs(Ui) @ np.abs(Uj).T + abs(math.log2(sf2))) + 4 * EPS


LD = np.longdouble
LD_OK = np.finfo(LD).nmant >= 63          # x86-64: 64-bit significand, 2^-11 of float64's rounding


def t_exact(Xi, Xj, ell, sf):
    """log2 sf^2 - log2(e)/2 |(x_i - x_j)/ell|^2 by direct differences in long double: its error is about 2^-11 of the
    kernels' bounds, so those bounds hold against it unchanged."""
    D = (Xi.astype(LD)[:, None, :] - Xj.astype(LD)[None, :, :]) / np.asarray(ell, dtype=LD)
    return 2 * np.log2(abs(LD(sf))) - (LD(0.5) / np.log(LD(2))) * np.einsum('ijd,ijd->ij', D, D)


def k_exact(t):
    """2^t in long double (no underflow down to 2^-16382)."""
    return np.exp2(np.asarray(t, dtype=LD))


def ks_t(X, Z, ell, sf2):
    """The ks kernel's te (numpy order, no fma) and its bound: (te, bound), shape (N, H)."""
    ie = 1.0 / ell
    xs = X * ie
    zs = Z * ie
    df = xs[:, None, :] - zs[None, :, :]
    dist = np.einsum('ijd,ijd->ij', df, df)
    te = -HALF_LOG2E * dist + math.log2(sf2)
    return te, ks_bound(xs, zs, df, dist, te)


def ks_bound(xs, zs, df, dist, te):
    Nx = xs.shape[1]
    ur = EPS / 2
    ad = np.abs(df)
    a = 2 * ur * (np.abs(xs)[:, None, :] + np.abs(zs)[None, :, :]) + 2 * ur * ad
    return HALF_LOG2E * (2 * np.einsum('ijd,ijd->ij', ad, a) + (Nx / 2 + 3) * EPS * dist) + EPS * np.abs(te) + 4 * EPS


def rel_bound(dt):
    """Relative error of one entry 2^t~ against 2^t* given |t~ - t*| <= dt."""
    return EXP2_ULP * EPS + np.expm1(math.log(2.0) * np.asarray(dt))

"""The device roll-outs (gpmpc_rollout_batch, gpmpc_rollout_batch_grad and gpmpc_rollout_sample) against the
long-double restatement oracle/rollout_oracle_ld.py fed the engine's own alpha and L^-1, at every shape their kernels
branch on (CASES, SAMPLE_CASES: the comment of each names the branch).  At every shape gpmpc_rollout_batch must give
gpmpc_rollout_batch_grad's means, vars and cov_last bit for bit (it skips the derivative chain and its buffers), and a
trajectory run alone must give its row of the batch bit for bit, for every output of all three entry points.

Errors are normalised entry by entry by the sums of |terms| the reference carries through the steps, so cond(K) enters
neither side.  Before any comparison the guards require every tangent column class (z0, U rows, K entries) and every
block of Sigma (xu, ux, uu, as rollout_feedback_kernel writes them) and of its tangent dS (xx, xu, ux, uu) to move some
output by at least GUARD x the bar x its normaliser, so a degenerate problem cannot hide a dropped term.  Nt <= 6 keeps
the rounding propagated through the recursion far below the bars; with 'ME' the reference is also fed the engine's own
means (predict_core's ME never reads Sigma, so that check has no propagation at all).

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, largest normalised error over every case and call (case):

    mean 7.4e-17 (auto_nx32)   var 5.7e-18 (auto_nx32)   cov_last 5.7e-18 (auto_nx32)   dmean 1.2e-16 (auto_nx32)
    dvar 1.9e-17 (ny16_nu16)   samples 2.9e-17 (s_b130)

TOL is 10x each maximum rounded up in its first digit.  The smallest guard ratios: a column class moves its dmean or
dvar by >= 3.0e-9 of the normaliser (n1100, against GUARD x TOL <= 2e-11); a dropped Sigma or dS block moves some
output by >= 3.9e6 x its bar (n1100).  Every keep decision of the sample cases is decisive or a clear drop, so
every kept flag is compared: the cases end before a sampled path revisits its inputs so closely that its conditional
variances sit at rounding level near DELTA sf2 (a closed loop of 12 steps left 42 of 144 such decisions).
"""
import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from oracle.rollout_oracle_ld import DS_BLOCKS, LD, MARGIN, SIGMA_BLOCKS, rollout_ld, sample_ld
from tests._util import normalised

pytestmark = pytest.mark.gpu

# name -> (N, Nx, Ny, Nu, B, Nt, options); options: 'scale' (a normalised GP's [sY | mY | mX | sX]), with feedback
# 'uscale' and 'xref'.  The tangent kernel runs 8 warps, one parameter column each, P = Nx + (Nt-1) Nu open loop or
# Nx + Nu Ny with K; the feedback kernel strides 256 threads over Nu Ny and Nx^2; the derivative chain picks NXP 8 / 16
# / 32 from Nx and runs GR_CHUNK = 1024-point blocks over Npad; predict passes run in HB = 64-point chunks of B.
CASES = {
    'p4': (200, 3, 2, 1, 3, 2, ()),                    # P = 4 open loop, 5 with K: idle warps; Ny 2
    'ny1_nu4': (200, 5, 1, 4, 2, 5, ('scale',)),       # a 1x1 cov; K (4x1) is a column; P = 9 with K
    'nx9': (300, 9, 5, 4, 2, 4, ('scale', 'uscale')),  # NXP 16 at its bottom
    'nx17': (300, 17, 9, 8, 1, 3, ('xref',)),          # NXP 32 at its bottom; B 1
    'ny31_nu1': (300, 32, 31, 1, 1, 3, ()),            # Nx 32 with one input: per-warp tangent block 2016 doubles; NXP 32
    'ny16_nu16': (300, 32, 16, 16, 1, 3, ('scale', 'uscale', 'xref')),   # Nu Ny = 256: one full stride; P = 288
    'nu_gt_ny': (200, 7, 2, 5, 2, 5, ('uscale', 'xref')),   # dS_uu's dK C K^T, K C dK^T with ki in 0..4, kk in 0..1
    'auto': (200, 3, 3, 0, 2, 5, ('scale',)),          # Nu 0: no input blocks, P = Nx
    'auto_nx32': (200, 32, 32, 0, 2, 3, ()),           # Ny = Nx = 32: the largest tangent layout (per warp 2112 doubles,
                                                       # 143,616 B in all), the one smem_opt_in sizes; P = 32 = 4 rounds
    'b64': (150, 4, 2, 2, 64, 3, ()),                  # one full HB chunk
    'b65': (150, 4, 2, 2, 65, 3, ('scale',)),          # HB chunks of 64 and 1
    'b130': (150, 4, 2, 2, 130, 3, ('scale', 'uscale', 'xref')),   # HB chunks of 64, 64 and 2
    'n1100': (1100, 10, 6, 4, 2, 4, ()),               # Npad 1152: two GR_CHUNK blocks (1024 and 76 points); NXP 16
}
# name -> (N, Nx, Ny, Nu, B, Nt, options); 'xi' process noise, 'fb' feedback, 'drop' a forced drop.  sample_cond_kernel:
# 8 warps over the kept points (j += 8), lanes < Nx form the input differences, solve_rows runs HB chunks of B.
SAMPLE_CASES = {
    's_nx32': (200, 32, 2, 30, 3, 14, ('xi',)),        # Nx 32: every lane a difference; up to 14 kept points (> 8)
    's_b130': (150, 5, 3, 2, 130, 12, ('scale',)),     # Ny 3 at B 130: solve_rows in chunks of 64, 64 and 2
    's_b130_xi': (150, 5, 3, 2, 130, 12, ('xi',)),     # the same with process noise
    's_fb': (200, 6, 3, 3, 4, 7, ('fb', 'scale', 'uscale', 'xref', 'xi')),    # inputs from the sampled state; Nt 7
                                                       # ends before the closed loop's variances reach rounding level
    's_drop': (100, 3, 2, 1, 4, 10, ('drop',)),        # steps 2..7 repeat step 1's input: dropped; steps 8, 9 kept
}
KEYS = ('mean', 'var', 'cov_last', 'dmean', 'dvar')
# bars on the largest error normalised by the sum of |terms| (measured maxima in the module docstring)
TOL = dict(mean=8e-16, var=6e-17, cov_last=6e-17, dmean=2e-15, dvar=2e-16, samples=3e-16)
GUARD = 1e4


def _problem(N, Nx, Ny, Nu, B, Nt, opts, seed):
    """Engine (factorised), X, hyper, alpha, L^-1 (long double) and the roll-out arguments of one case."""
    import gp_mpc_b200
    p = orc.synthetic_problem(N, Nx, Ny, config_id=900 + Nx + Ny, H=1)
    p['hyper'][:, Nx + 1] = 0.1                      # variances well above sn^2 = 1e-4, so their derivatives pass the guards
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
    eng.set_data(p['X'], p['Y'])
    eng.set_hyper(p['hyper'])
    assert not eng.factorize().any()
    alpha = np.stack([eng.get(L.GET_ALPHA, a) for a in range(Ny)])
    linv = np.stack([eng.get(L.GET_LINV, a) for a in range(Ny)]).astype(LD)
    rng = np.random.default_rng(seed + Nx)
    z0 = 0.5 * rng.standard_normal((B, Nx))
    U = 0.5 * rng.standard_normal((B, Nt, Nu))
    A = rng.standard_normal((Nx, Nx))
    S0 = 1e-3 * (A @ A.T / Nx + np.eye(Nx))
    S0 = np.stack([S0 * (1 + 0.1 * b) for b in range(B)])
    arg = dict(scale=None, K=None, x_ref=None, uscale=None)
    if 'scale' in opts:
        arg['scale'] = np.stack([rng.uniform(0.5, 1.5, Ny), 0.1 * rng.standard_normal(Ny),
                                 0.1 * rng.standard_normal(Ny), rng.uniform(0.5, 1.5, Ny)])
    if Nu:
        arg['K'] = 0.5 * rng.standard_normal((Nu, Ny)) / np.sqrt(Ny)
        if 'uscale' in opts:
            arg['uscale'] = np.stack([0.1 * rng.standard_normal(Nu), rng.uniform(0.5, 1.5, Nu)])
        if 'xref' in opts:
            arg['x_ref'] = 0.2 * rng.standard_normal(Ny)
    return eng, p['X'], p['hyper'], alpha, linv, z0, U, S0, arg


def _ratio(part, scale):
    return float(np.max(np.abs(part) / np.where(scale > 0, scale, np.inf), initial=0.0))


def check_guards(ld_args, ref, meth, fb, Nx, Ny, Nu, Nt):
    """Every column class of the tangents and (TA) every Sigma / dS block moves some output by >= GUARD x the bar x the
    normaliser.  Returns the smallest ratio per guard."""
    seen = {}
    cls = {'z0': slice(0, Nx)}
    if Nu:
        cls['K' if fb else 'U'] = slice(Nx, None)
    for c, sl in cls.items():
        if c == 'U' and Nt < 2:
            continue
        for k in ('dmean', 'dvar'):
            r = _ratio(ref[k][..., sl], ref['s_' + k][..., sl])
            assert r >= GUARD * TOL[k], ('column class', c, k, r)
            seen['%s %s' % (c, k)] = r
    if meth == 'TA' and Nt > 1:
        names = (SIGMA_BLOCKS + DS_BLOCKS) if fb else ('xx',)
        for name in names:
            d = rollout_ld(*ld_args, tangents=True, drop=(name,))
            r = max(_ratio(ref[k] - d[k], ref['s_' + k]) / TOL[k] for k in KEYS)
            assert r >= GUARD, ('block', name, r)
            seen['block ' + name] = r
    return seen


def _alone_rows(B):
    """The trajectories run alone to check that their bits do not depend on the batch: the first, the last and the first
    of the second 64-point chunk."""
    return sorted({0, B - 1} | ({64} if B > 64 else set())) if B > 1 else []


def case_errors(name):
    """Per call ('TA', 'ME', 'ME fed', each open loop and with K): the largest normalised error of each output, after the
    guards (their smallest ratios under 'guards').  Asserts that gpmpc_rollout_batch gives the same means, vars and
    cov_last bits and that trajectories run alone give their rows' bits."""
    N, Nx, Ny, Nu, B, Nt, opts = CASES[name]
    eng, X, hyper, alpha, linv, z0, U, S0, arg = _problem(N, Nx, Ny, Nu, B, Nt, opts, 0)
    res = dict(guards={})
    for fb in ((False, True) if Nu else (False,)):
        kw = dict(arg) if fb else dict(arg, K=None, x_ref=None, uscale=None)
        for meth in ('TA', 'ME'):
            m = L.METHOD_TA if meth == 'TA' else L.METHOD_ME
            extra = (kw['scale'], kw['K'], kw['x_ref'], kw['uscale'])
            out = eng.rollout_batch_grad(z0, U, S0, m, *extra)
            plain = eng.rollout_batch(z0, U, S0, m, *extra)
            for k, x, y in zip(KEYS, plain, out):
                assert np.array_equal(x, y), (name, meth, fb, 'rollout_batch', k)
            for b in _alone_rows(B):
                sl = slice(b, b + 1)
                one = eng.rollout_batch_grad(z0[sl], U[sl], S0[sl], m, *extra)
                one_plain = eng.rollout_batch(z0[sl], U[sl], S0[sl], m, *extra)
                for k, x, y in zip(KEYS, one, out):
                    assert np.array_equal(x[0], y[b]), (name, meth, fb, 'alone', b, k)
                for k, x, y in zip(KEYS, one_plain, out):
                    assert np.array_equal(x[0], y[b]), (name, meth, fb, 'rollout_batch alone', b, k)
            got = dict(zip(KEYS, out))
            ld_args = (X, hyper, alpha, linv, z0, U, S0, meth, kw['scale'], kw['K'], kw['x_ref'], kw['uscale'])
            ref = rollout_ld(*ld_args, tangents=True)
            tag = '%s %s' % (meth, 'K' if fb else 'open')
            for g, r in check_guards(ld_args, ref, meth, fb, Nx, Ny, Nu, Nt).items():
                res['guards'][tag + ' ' + g] = r
            res[tag] = {k: normalised(got[k], ref[k], ref['s_' + k]) for k in KEYS}
            if meth == 'ME':
                fed = rollout_ld(*ld_args, tangents=True, means_in=got['mean'])
                res[tag + ' fed'] = {k: normalised(got[k], fed[k], fed['s_' + k]) for k in KEYS}
    eng.close()
    return res


@pytest.mark.parametrize('name', list(CASES))
def test_rollouts_vs_long_double(name):
    """means, vars, cov_last, dmeans and dvars of TA and ME, open loop and with feedback, against the reference within
    TOL of the sums of |terms|, after the guards."""
    res = case_errors(name)
    worst = {k: max(e[k] for c, e in res.items() if c != 'guards') for k in KEYS}
    print('[rollout] %s %s, smallest guard ratios: column class %.1e, block %.1e' % (
        name, ' '.join('%s %.1e' % kv for kv in worst.items()),
        min((r for g, r in res['guards'].items() if 'block' not in g), default=np.inf),
        min((r for g, r in res['guards'].items() if 'block' in g), default=np.inf)))
    for c, errs in res.items():
        if c == 'guards':
            continue
        bad = {k: e for k, e in errs.items() if not e <= TOL[k]}
        assert not bad, (name, c, bad)


def sample_errors(name):
    """(largest normalised sample error, number of unsure keep decisions, number of decisions, the engine's kept) of one
    sample case; asserts the kept flags of every decisive step and of every clear drop."""
    N, Nx, Ny, Nu, B, Nt, opts = SAMPLE_CASES[name]
    eng, X, hyper, alpha, linv, z0, U, _, arg = _problem(N, Nx, Ny, Nu, B, Nt, opts, 1)
    rng = np.random.default_rng(3)
    eps = rng.standard_normal((B, Nt, Ny))
    xi = rng.standard_normal((B, Nt, Ny)) if 'xi' in opts else None
    K = arg['K'] if 'fb' in opts else None
    scale = arg['scale']
    if 'drop' in opts:
        # sY = 0: every state input is (mY - mX) / sX whatever the sample, so with the input held the point repeats
        scale = np.stack([np.zeros(Ny), 0.3 * np.ones(Ny), np.zeros(Ny), np.ones(Ny)])
        U[:, 1:8] = U[:, 1:2]
        U[:, 8], U[:, 9] = U[:, 1] + 3.0, U[:, 1] - 3.0       # far from the held input and each other: kept
    extra = (scale, K, arg['x_ref'] if K is not None else None, arg['uscale'] if K is not None else None)
    samples, z_out, kept = eng.rollout_sample(z0, U, eps, xi, *extra)
    for b in _alone_rows(B):
        sl = slice(b, b + 1)
        one = eng.rollout_sample(z0[sl], U[sl], eps[sl], None if xi is None else xi[sl], *extra)
        for k, x, y in zip(('samples', 'z_out', 'kept'), one, (samples, z_out, kept)):
            assert np.array_equal(x[0], y[b]), (name, 'alone', b, k)
    eng.close()
    o = sample_ld(X, hyper, alpha, linv, z_out, eps, xi, kept=kept)
    err = normalised(samples, o['samples'], o['s_samples'])
    sure = o['margin'] >= MARGIN
    assert np.array_equal(kept[sure].astype(bool), o['kept'][sure]), name
    sf2 = (hyper[:, Nx] ** 2)[None, None, :]
    clear_drop = np.abs(np.asarray(o['d'], dtype=np.float64)) <= 0.1 * 1e-12 * sf2
    assert not kept[clear_drop].any(), name
    unsure = int(np.sum(~sure & ~clear_drop))
    return err, unsure, kept.size, kept


@pytest.mark.parametrize('name', list(SAMPLE_CASES))
def test_rollout_sample_vs_long_double(name):
    """Samples against sample_ld along the engine's own inputs and conditioning sets, within TOL of the sums of |terms|;
    every kept flag, each decision being either decisive (margin >= MARGIN) or a clear drop (|d| <= 0.1 DELTA sf2)."""
    err, unsure, n, kept = sample_errors(name)
    print('[sample] %s err %.1e, %d of %d keep decisions neither decisive nor a clear drop' % (name, err, unsure, n))
    assert err <= TOL['samples'], (name, err)
    assert unsure == 0, (name, unsure, n)
    opts = SAMPLE_CASES[name][6]
    assert kept[:, 0].all()
    if 'drop' in opts:
        assert not kept[:, 2:8].any() and kept[:, 8:].all()
    elif 'fb' not in opts:
        assert (kept.sum(1) > 8).any()              # the warp loop's second round

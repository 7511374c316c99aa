"""The device-pointer predict entry (gpmpc_predict_device, the call bench.py times) and the transports of the host entry
gpmpc_predict (gpmpc.cu:1668-1699).

gpmpc_predict moves its inputs [Z | Sigma] either by one H2D copy into dIn or by letting the ks kernel read them in place
from the mapped pinned buffer (zero-copy in), and its outputs either by the assembling CTA writing them straight into the
mapped buffer (zero-copy out) or by one D2H copy of the span [lo, hi) of dOut.  Both slabs are laid out by the handle's
capacity Hcap, which only grows, so the transport of a call depends on the handle's history as well as on the call.
The kernels behind every transport are the same and a fixed stream-K partition is bit-reproducible (DESIGN 4.5), so a
call must give the same bits through every transport and through gpmpc_predict_device; a float64 CPU oracle anchors the
values at the suite's 1e-6 gate.  `transport` below restates the selection; every case asserts the transport it is
meant to reach, so a change of thresholds fails a precondition instead of silently dropping a branch."""
import itertools
import threading

import numpy as np
import pytest

from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._engines import npad
from tests._util import relinf

TOL = 1e-6
HB = 64                                   # test points per predict pass (gpmpc.cu:23)
OUTPUTS = ('mean', 'var', 'cov', 'jac')


# ------------------------------------------------------------------ transport model (no GPU)
def ks_chunk(npad, nloc, Nx):
    """gpmpc.cu:807-811."""
    if npad < 8192:
        return 128
    return 1024 if (nloc >= 2 and Nx <= 12) else 512


def ks_blocks(npad, nloc, Nx):
    """gpmpc.cu:814."""
    return -(-npad // ks_chunk(npad, nloc, Nx))


def grow(hcap, H):
    """ensure_predict_bufs (gpmpc.cu:841-855): the layout of dIn / dOut is redone for max(H, 64) points when H exceeds
    the capacity; it never shrinks.  hcap = 0 on a handle that has not predicted yet."""
    return max(H, HB) if H > hcap else hcap


def transport(npad, nloc, Nx, Ny, H, hcap, has_sigma, spp, outputs=OUTPUTS):
    """(zc_in, zc_out) of gpmpc_predict (gpmpc.cu:1668-1690) for a call of H points on a handle of nloc outputs whose
    capacity was hcap before the call.  has_sigma: a TA call that passes Sigma (ME never copies it); outputs: the
    non-NULL ones among mean / var / cov / jac."""
    cap = grow(hcap, H)
    ns = (H if spp else 1) * Nx * Nx if has_sigma else 0
    in_span = cap * Nx + ns if ns else H * Nx
    off = dict(mean=0, var=cap * Ny, jac=2 * cap * Ny, cov=2 * cap * Ny + cap * Ny * Nx)
    size = dict(mean=H * Ny, var=H * Ny, jac=H * Ny * Nx, cov=H * Ny * Ny)
    out_span = (max(off[o] + size[o] for o in outputs) - min(off[o] for o in outputs)) if outputs else 0
    ks_ctas = ks_blocks(npad, nloc, Nx) * (-(-min(H, HB) // 8) * 8) * nloc
    zc_in = H <= HB and ks_ctas * Nx * 8 <= 256 * 1024 and in_span * 8 <= 64 * 1024
    zc_out = out_span * 8 <= 1024 * 1024
    return zc_in, zc_out


# C. one shape per (zc_in, zc_out): name -> (N, Nx, Ny, H)
SHAPES = {(1, 1): (300, 5, 3, 20),          # small problem
          (0, 1): (300, 6, 4, 65),          # one point past a chunk: dIn, outputs still small
          (0, 0): (700, 10, 8, 2100),       # > 1 MiB of outputs; assemble_kernel's grid-stride loop (H > 2048)
          (1, 0): (120, 10, 40, 64)}        # 40 outputs: > 1 MiB of outputs while the inputs still fit zero-copy
# D. a small TA call before and after one call of H_BIG points on the same handle
HIST = (300, 10, 8, 20)
H_BIG = 2100


def test_transport_model_reaches_every_branch():
    """The shapes of C land on their four (zc_in, zc_out) pairs for TA with one Sigma, TA with a Sigma per point and ME
    on a fresh handle; D's small call switches from zero-copy to copies in both directions once the handle has held
    2100 points (in_span 21100 doubles, out_span 202880: about 169 KB in and 1.6 MB out per call); B's copy-out shape
    copies out for some output subsets with mean NULL, so the D2H source offset lo is not 0."""
    for want, (N, Nx, Ny, H) in SHAPES.items():
        for has_sigma, spp in ((True, 0), (True, 1), (False, 0)):
            assert transport(npad(N), Ny, Nx, Ny, H, 0, has_sigma, spp) == want, (want, has_sigma, spp)
            assert transport(npad(N), Ny, Nx, Ny, H, grow(0, H), has_sigma, spp) == want
    N, Nx, Ny, H = HIST
    assert transport(npad(N), Ny, Nx, Ny, H, 0, True, 0) == (1, 1)
    assert grow(grow(0, H), H_BIG) == H_BIG
    assert transport(npad(N), Ny, Nx, Ny, H, H_BIG, True, 0) == (0, 0)
    assert transport(npad(N), Ny, Nx, Ny, H_BIG, 0, True, 0) == (0, 0)
    N, Nx, Ny, H = SHAPES[(0, 0)]
    outs = [s for s in _subsets() if not transport(npad(N), Ny, Nx, Ny, H, H, True, 0, s)[1]]
    assert ('jac',) in outs and ('var', 'cov') in outs and ('cov',) in outs and ('mean',) not in outs
    N, Nx, Ny, H = SHAPES[(1, 1)]
    assert all(transport(npad(N), Ny, Nx, Ny, H, 64, True, 0, s) == (1, 1) for s in _subsets())
    # the C5 headline shape: copy in (the ks grid re-reads Z too often for zero-copy), zero-copy out
    assert transport(16384, 8, 10, 8, 50, 0, True, 0) == (0, 1)


def _subsets():
    return [s for r in range(1, 5) for s in itertools.combinations(OUTPUTS, r)]


# ------------------------------------------------------------------ GPU helpers
def _ptr(t):
    return None if t is None else t.data_ptr()


class Model:
    """A factorised handle on a seeded synthetic problem with every output, the capacity its calls have grown it to,
    and the float64 oracle of its predictions (independent CPU factors)."""

    def __init__(self, N, Nx, Ny, config_id, X=None, Y=None, hyper=None):
        import gp_mpc_b200
        if X is None:
            p = orc.synthetic_problem(N, Nx, Ny, config_id=config_id)
            X, Y, hyper = p['X'], p['Y'], p['hyper']
        self.X, self.Y, self.hyper = X, Y, hyper
        self.N, self.Nx, self.Ny = N, Nx, Ny
        self.rng = np.random.default_rng(config_id)
        self.eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
        self.eng.set_data(X, Y)
        self.eng.set_hyper(hyper)
        assert not self.eng.factorize().any()
        self.hcap = 0
        self._fac = None

    def close(self):
        self.eng.close()

    def transport(self, H, has_sigma, spp, outputs=OUTPUTS):
        return transport(npad(self.N), self.Ny, self.Nx, self.Ny, H, self.hcap, has_sigma, spp, outputs)

    def inputs(self, H, spp):
        """Distinct test points and input covariances: (Z (H,Nx), Sigma (Nx,Nx) or (H,Nx,Nx))."""
        Nx = self.Nx
        Z = 0.5 * self.rng.standard_normal((H, Nx))
        A = self.rng.standard_normal((H if spp else 1, Nx, Nx))
        S = 1e-4 * np.eye(Nx) + 1e-5 * A @ A.transpose(0, 2, 1)
        return Z, (S if spp else S[0])

    def host(self, Z, Sigma, method, want_cov=True, want_jac=True):
        self.hcap = grow(self.hcap, Z.shape[0])
        return self.eng.predict(Z, Sigma, method, want_cov=want_cov, want_jac=want_jac)

    def device(self, Z, Sigma, method, outs=None, sync=True):
        """gpmpc_predict_device on torch tensors.  outs: name -> device tensor or None (default: all four, fresh).
        Returns the output tensors; with sync=False the caller synchronises the handle before reading them."""
        import torch
        H, Ny, Nx = Z.shape[0], self.Ny, self.Nx
        if outs is None:
            outs = dict(mean=torch.empty(H, Ny, dtype=torch.float64, device='cuda'),
                        var=torch.empty(H, Ny, dtype=torch.float64, device='cuda'),
                        cov=torch.empty(H, Ny, Ny, dtype=torch.float64, device='cuda'),
                        jac=torch.empty(H, Ny, Nx, dtype=torch.float64, device='cuda'))
        dZ = Z if torch.is_tensor(Z) else torch.from_numpy(np.ascontiguousarray(Z)).cuda()
        dS = Sigma if (Sigma is None or torch.is_tensor(Sigma)) else torch.from_numpy(np.ascontiguousarray(Sigma)).cuda()
        spp = int(dS is not None and dS.dim() == 3)
        # the copies run on torch's stream and the handle's stream does not wait for it; a stream sync, not a device
        # sync, so calls already enqueued on the handle keep running
        torch.cuda.current_stream().synchronize()
        self.hcap = grow(self.hcap, H)
        self.eng.predict_device(method, H, dZ.data_ptr(), _ptr(dS), spp, *[_ptr(outs.get(k)) for k in OUTPUTS],
                                sync=sync)
        outs = dict(outs)
        outs['_keep'] = (dZ, dS)                  # alive until the caller has synchronised
        return outs

    def factors(self):
        if self._fac is None:
            fs = [orc.factor_large(self.X, self.Y[:, a], self.hyper[a]) for a in range(self.Ny)]
            assert not any(f['jitter'] for f in fs)
            self._fac = (np.stack([f['alpha'] for f in fs]), np.stack([f['chol'] for f in fs]))
        return self._fac

    def oracle(self, Z, Sigma, method):
        alpha, chol = self.factors()
        mo, vo = orc.gp_mean_var(self.X, self.hyper, alpha, chol, Z)
        Jo = orc.gp_mean_jac(self.X, self.hyper, alpha, Z)
        co = orc.ta_cov(vo, Jo, Sigma) if method == L.METHOD_TA else orc.me_cov(vo)
        return dict(mean=mo, var=vo, cov=co, jac=Jo)


def _np(outs):
    return {k: (None if outs.get(k) is None else outs[k].cpu().numpy()) for k in OUTPUTS}


def _same(a, b, names=OUTPUTS):
    for k in names:
        assert np.array_equal(a[k], b[k]), k


def _close(got, ref, names=OUTPUTS):
    for k in names:
        assert relinf(got[k], ref[k]) < TOL, (k, relinf(got[k], ref[k]))


def _as_dict(t):
    return dict(zip(OUTPUTS, t))


# ------------------------------------------------------------------ A. gpmpc_predict_device at bench.py's inputs
def _bench_model(name):
    from bench import WORKLOADS, make_workload
    wl = WORKLOADS[name]
    N, Nx, Ny, H = wl['N'], wl['Nx'], wl['Ny'], wl['H']
    w = make_workload(N, Nx, Ny, wl['cfg'], H)
    return Model(N, Nx, Ny, wl['cfg'], X=w['X'], Y=w['Y'], hyper=w['hyper']), w


def _bench_step(m, w):
    """bench.py's timed step: TA, one Sigma (spp = 0), device outputs, sync = False, then one synchronize."""
    import torch
    outs = m.device(torch.from_numpy(w['Z']).cuda(), torch.from_numpy(w['Sigma']).cuda(), L.METHOD_TA, sync=False)
    m.eng.synchronize()
    return _np(outs)


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['c2', 'c3'])
def test_bench_step_vs_oracle(name):
    """The outputs of bench.py's timed call at C2 (N=1000) and C3 (N=4096), every output against independent CPU factors
    (factor_large / predict_large / ta_cov), and bit for bit against gpmpc_predict on the same handle."""
    m, w = _bench_model(name)
    Ny, Nx, H = m.Ny, m.Nx, w['Z'].shape[0]
    got = _bench_step(m, w)
    mo = np.zeros((H, Ny)); vo = np.zeros((H, Ny)); Jo = np.zeros((H, Ny, Nx))
    for a in range(Ny):
        f = orc.factor_large(m.X, m.Y[:, a], m.hyper[a])
        assert not f['jitter']
        mo[:, a], vo[:, a], Jo[:, a] = orc.predict_large(m.X, m.hyper[a], f['alpha'], f['chol'], w['Z'])
        del f
    _close(got, dict(mean=mo, var=vo, jac=Jo, cov=orc.ta_cov(vo, Jo, w['Sigma'])))
    _same(got, _as_dict(m.host(w['Z'], w['Sigma'], L.METHOD_TA)))
    m.close()


@pytest.mark.gpu
def test_bench_step_c5():
    """C5 (N=16384, Nx=10, Ny=8, all outputs on one handle as at --gpus 1): the timed call's outputs are gpmpc_predict's
    bits for all 8 outputs, and output Ny-1 matches an independent CPU factor at 1e-6 (bench.py's own parity check
    compares the separate e2e call)."""
    m, w = _bench_model('c5')
    Ny = m.Ny
    got = _bench_step(m, w)
    again = _bench_step(m, w)
    _same(got, again)
    host = _as_dict(m.host(w['Z'], w['Sigma'], L.METHOD_TA))
    _same(got, host)
    a = Ny - 1
    f = orc.factor_large(m.X, m.Y[:, a], m.hyper[a])
    assert not f['jitter']
    mo, vo, Jo = orc.predict_large(m.X, m.hyper[a], f['alpha'], f['chol'], w['Z'])
    del f
    m.close()
    assert relinf(got['mean'][:, a], mo) < TOL and relinf(got['var'][:, a], vo) < TOL
    assert relinf(got['jac'][:, a], Jo) < TOL
    assert relinf(got['cov'][:, a, a], orc.ta_cov(vo[:, None], Jo[:, None, :], w['Sigma'])[:, 0, 0]) < TOL


@pytest.mark.gpu
def test_device_entry_sigma_per_point_me_and_no_sigma():
    """gpmpc_predict_device with one Sigma per point, with ME and dSigma = NULL, and with TA, d_cov = NULL and
    dSigma = NULL (allowed: only a covariance output needs Sigma, gpmpc.cu:1496): the oracle at 1e-6 and
    gpmpc_predict's bits."""
    m = Model(300, 6, 3, config_id=11)
    Z, Sg = m.inputs(30, spp=1)
    got = _np(m.device(Z, Sg, L.METHOD_TA))
    _close(got, m.oracle(Z, Sg, L.METHOD_TA))
    _same(got, _as_dict(m.host(Z, Sg, L.METHOD_TA)))
    got = _np(m.device(Z, None, L.METHOD_ME))
    _close(got, m.oracle(Z, None, L.METHOD_ME))
    _same(got, _as_dict(m.host(Z, None, L.METHOD_ME)))
    import torch
    outs = dict(mean=torch.empty(30, 3, dtype=torch.float64, device='cuda'),
                var=torch.empty(30, 3, dtype=torch.float64, device='cuda'),
                jac=torch.empty(30, 3, 6, dtype=torch.float64, device='cuda'))
    got = _np(m.device(Z, None, L.METHOD_TA, outs=outs))
    _close(got, m.oracle(Z, Sg, L.METHOD_TA), ('mean', 'var', 'jac'))
    _same(got, _as_dict(m.host(Z, None, L.METHOD_TA, want_cov=False)), ('mean', 'var', 'jac'))
    m.close()


# ------------------------------------------------------------------ B. output regions are exact
PAD = 5                                      # odd: every output starts at an odd element offset


def _shape(name, H, Ny, Nx):
    return dict(mean=(H, Ny), var=(H, Ny), cov=(H, Ny, Ny), jac=(H, Ny, Nx))[name]


@pytest.mark.gpu
def test_device_outputs_stay_in_their_regions():
    """gpmpc_predict_device writing into slices at odd element offsets of NaN-filled buffers, at H = 20 (the fused
    assembly) and H = 2100 (assemble_kernel): the plain call's bits inside, the sentinels untouched outside."""
    import torch
    m = Model(*SHAPES[(0, 0)][:3], config_id=12)
    for H in (20, H_BIG):
        Z, S = m.inputs(H, spp=0)
        ref = _np(m.device(Z, S, L.METHOD_TA))
        bufs, outs = {}, {}
        for k in OUTPUTS:
            shp = _shape(k, H, m.Ny, m.Nx)
            n = int(np.prod(shp))
            bufs[k] = torch.full((n + 2 * PAD,), float('nan'), dtype=torch.float64, device='cuda')
            outs[k] = bufs[k][PAD:PAD + n].view(shp)
            assert outs[k].data_ptr() % 16 == 8          # odd element offset of a 16-byte aligned allocation
        got = _np(m.device(Z, S, L.METHOD_TA, outs=outs))
        _same(got, ref)
        for k in OUTPUTS:
            b = bufs[k].cpu().numpy()
            assert np.isnan(b[:PAD]).all() and np.isnan(b[-PAD:]).all(), k
    m.close()


def _host_call(m, method, Z, Sigma, names):
    """gpmpc_predict through ctypes into caller-side buffers at odd offsets of NaN-filled arrays; NULL for the outputs
    not in names.  Returns (rc, outputs, buffers)."""
    lib = L.load()
    H = Z.shape[0]
    Z = np.ascontiguousarray(Z)
    S = None if Sigma is None else np.ascontiguousarray(Sigma)
    spp = int(S is not None and S.ndim == 3)
    bufs, outs, ptrs = {}, {}, []
    for k in OUTPUTS:
        if k in names:
            shp = _shape(k, H, m.Ny, m.Nx)
            n = int(np.prod(shp))
            bufs[k] = np.full(n + 2 * PAD, np.nan)
            outs[k] = bufs[k][PAD:PAD + n].reshape(shp)
            ptrs.append(outs[k].ctypes.data_as(L._dp))
        else:
            ptrs.append(None)
    m.hcap = grow(m.hcap, H)
    rc = lib.gpmpc_predict(m.eng.h, method, H, Z.ctypes.data_as(L._dp), None if S is None else S.ctypes.data_as(L._dp),
                           spp, ptrs[0], ptrs[1], ptrs[2], ptrs[3])
    return rc, outs, bufs


@pytest.mark.gpu
@pytest.mark.parametrize('want', [(1, 1), (0, 0)])
def test_host_output_subsets(want):
    """gpmpc_predict with every non-empty subset of {mean, var, cov, jac} (NULL for the rest) into caller buffers at
    odd offsets inside NaN sentinels, on a zero-copy shape and on the copy-out shape: each output is the full call's,
    bit for bit, and nothing outside it is written.  The subsets move lo, the first output of the D2H span; on the
    copy-out shape jac, cov and (var, cov) copy out with mean NULL.  The call with every output NULL returns OK."""
    N, Nx, Ny, H = SHAPES[want]
    m = Model(N, Nx, Ny, config_id=13)
    Z, S = m.inputs(H, spp=0)
    ref = _as_dict(m.host(Z, S, L.METHOD_TA))
    seen = set()
    for names in _subsets():
        tr = m.transport(H, True, 0, names)
        seen.add((tr[1], 'mean' in names))
        rc, outs, bufs = _host_call(m, L.METHOD_TA, Z, S, names)
        assert rc == L.OK, (names, m.eng.lib.gpmpc_last_error(m.eng.h))
        for k in names:
            assert np.array_equal(outs[k], ref[k]), (names, k, tr)
            assert np.isnan(bufs[k][:PAD]).all() and np.isnan(bufs[k][-PAD:]).all(), (names, k)
    rc, _, _ = _host_call(m, L.METHOD_TA, Z, S, ())
    assert rc == L.OK
    if want == (1, 1):
        assert seen == {(True, True), (True, False)}
    else:
        assert (False, False) in seen and (False, True) in seen and (True, True) in seen
    m.close()


# ------------------------------------------------------------------ C. the four transports
@pytest.mark.gpu
@pytest.mark.parametrize('want', list(SHAPES))
def test_transports_agree_bit_for_bit(want):
    """On the shape of each (zc_in, zc_out): gpmpc_predict and gpmpc_predict_device give the same bits for TA with one
    Sigma, TA with a Sigma per point and ME, and both match the oracle (gp_mean_var / gp_mean_jac / ta_cov) at 1e-6.
    The device entry reads and writes device memory directly, so it is the common reference of all four transports."""
    N, Nx, Ny, H = SHAPES[want]
    m = Model(N, Nx, Ny, config_id=14 + N)
    for method, spp in ((L.METHOD_TA, 0), (L.METHOD_TA, 1), (L.METHOD_ME, 0)):
        Z, S = m.inputs(H, spp)
        Sig = S if method == L.METHOD_TA else None
        assert m.transport(H, Sig is not None, spp) == want
        host = _as_dict(m.host(Z, Sig, method))
        dev = _np(m.device(Z, Sig, method))
        _same(host, dev)
        _close(host, m.oracle(Z, S, method))
    m.close()


# ------------------------------------------------------------------ D. history
@pytest.mark.gpu
def test_small_call_after_a_large_one():
    """A small TA call on a fresh handle goes zero-copy both ways; after one call of 2100 points the same call copies
    both ways (the capacity-based layout, DESIGN 7).  The two small calls give the same bits, and the large call matches
    the oracle."""
    N, Nx, Ny, H = HIST
    m = Model(N, Nx, Ny, config_id=15)
    Z, S = m.inputs(H, spp=0)
    assert m.transport(H, True, 0) == (1, 1)
    first = _as_dict(m.host(Z, S, L.METHOD_TA))
    Zb, Sb = m.inputs(H_BIG, spp=1)
    assert m.transport(H_BIG, True, 1) == (0, 0)
    big = _as_dict(m.host(Zb, Sb, L.METHOD_TA))
    assert m.hcap == H_BIG
    assert m.transport(H, True, 0) == (0, 0)
    second = _as_dict(m.host(Z, S, L.METHOD_TA))
    _same(first, second)
    _close(first, m.oracle(Z, S, L.METHOD_TA))
    _close(big, m.oracle(Zb, Sb, L.METHOD_TA))
    m.close()


# ------------------------------------------------------------------ E. back to back, no host sync
SEQ_H = (50, 1, 64, 65, 130, 7, 2100, 50)


def _sequence(m, host_at=None):
    """SEQ_H enqueued through gpmpc_predict_device with no sync in between: TA and ME alternate, the TA calls alternate
    one Sigma and a Sigma per point, each call has its own Z and outputs, predict_ctas changes (dPart grows) after the
    fourth call and H = 2100 grows the gather buffer dG while earlier calls may still run.  host_at: index of a host
    gpmpc_predict call placed before that device call.  Returns [(H, method, Z, S, ctas, outputs)]."""
    import torch
    calls = []
    big_ctas = 4 * torch.cuda.get_device_properties(0).multi_processor_count + 8    # above the default grid
    m.eng.set_option('predict_ctas', 0)
    for i, H in enumerate(SEQ_H):
        if i == 4:
            m.eng.set_option('predict_ctas', big_ctas)
        ctas = big_ctas if i >= 4 else 0
        if i == host_at:
            Zh, Sh = m.inputs(40, spp=1)
            calls.append((40, L.METHOD_TA, Zh, Sh, ctas, _as_dict(m.host(Zh, Sh, L.METHOD_TA)), 'host'))
        method = L.METHOD_TA if i % 2 == 0 else L.METHOD_ME
        Z, S = m.inputs(H, spp=(i // 2) % 2)
        Sig = S if method == L.METHOD_TA else None
        calls.append((H, method, Z, Sig, ctas, m.device(Z, Sig, method, sync=False), 'device'))
    m.eng.synchronize()
    return calls


def _replay(m, calls):
    for H, method, Z, S, ctas, outs, kind in calls:
        m.eng.set_option('predict_ctas', ctas)
        got = outs if kind == 'host' else _np(outs)
        again = _as_dict(m.host(Z, S, method)) if kind == 'host' else _np(m.device(Z, S, method, sync=True))
        _same(got, again)


@pytest.mark.gpu
def test_back_to_back_without_sync():
    """Each call of a sequence enqueued without host sync equals the same call made alone afterwards (sync = True), bit
    for bit: the stream-K counters clean themselves and buffer growth waits for the calls in flight.  Then again with a
    host gpmpc_predict in the middle of the sequence.  The first sequence is also checked against the oracle."""
    m = Model(300, 10, 8, config_id=16)
    calls = _sequence(m)
    _replay(m, calls)
    for H, method, Z, S, ctas, outs, kind in calls:
        _close(_np(outs), m.oracle(Z, S, method))
    calls = _sequence(m, host_at=3)
    assert sum(c[-1] == 'host' for c in calls) == 1
    _replay(m, calls)
    m.close()


# ------------------------------------------------------------------ F. two handles, two host threads
def _mixed_calls(m, n=20):
    out = []
    for i in range(n):
        H = (5, 64, 70, 33)[i % 4]
        Z, S = m.inputs(H, spp=i % 3 == 0)
        out.append((Z, S, L.METHOD_TA if i % 2 == 0 else L.METHOD_ME, 'device' if i % 4 in (1, 2) else 'host'))
    return out


def _run_calls(m, calls, results, barrier=None):
    import torch
    ta = L.METHOD_TA
    try:
        dev = []
        for Z, S, method, kind in calls:          # device copies of the inputs, made before the threads meet
            dev.append((torch.from_numpy(Z).cuda(), torch.from_numpy(S).cuda() if method == ta else None))
        torch.cuda.current_stream().synchronize()
        if barrier is not None:
            barrier.wait()
        for (Z, S, method, kind), (dZ, dS) in zip(calls, dev):
            if kind == 'host':
                results.append(_as_dict(m.host(Z, S if method == ta else None, method)))
            else:
                results.append(_np(m.device(dZ, dS, method, sync=True)))
    except BaseException as e:                     # re-raised by the main thread
        if barrier is not None:
            barrier.abort()
        results.append(e)


@pytest.mark.gpu
def test_two_handles_two_threads():
    """Two handles with different models on device 0, each driven by its own host thread with 20 calls that mix
    gpmpc_predict and gpmpc_predict_device: every result equals the same call made with the two handles used one after
    the other."""
    ma = Model(300, 6, 3, config_id=17)
    mb = Model(500, 8, 5, config_id=18)
    ca, cb = _mixed_calls(ma), _mixed_calls(mb)
    seq_a, seq_b = [], []
    _run_calls(ma, ca, seq_a)
    _run_calls(mb, cb, seq_b)
    for r in seq_a + seq_b:
        if isinstance(r, BaseException):
            raise r
    par_a, par_b = [], []
    barrier = threading.Barrier(2)
    ts = [threading.Thread(target=_run_calls, args=(ma, ca, par_a, barrier)),
          threading.Thread(target=_run_calls, args=(mb, cb, par_b, barrier))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    for r in par_a + par_b:
        if isinstance(r, BaseException):
            raise r
    assert len(par_a) == len(seq_a) == len(ca) and len(par_b) == len(seq_b) == len(cb)
    for x, y in zip(par_a + par_b, seq_a + seq_b):
        _same(x, y)
    ma.close(); mb.close()

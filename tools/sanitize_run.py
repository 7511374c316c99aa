"""Small end-to-end pass over every kernel of the engine for compute-sanitizer
(memcheck / racecheck / synccheck / initcheck):  K build, leaf + DMMA GEMMs (cp.async feeds; the TMA
tensor-map feed on a second, 24-output handle), alpha, NLML + gradient, the persistent stream-K predict kernel with tile
fix-ups (several grid sizes, lower and upper mode), gpmpc_predict_device, gpmpc_predict's copy transports, predict_grad, EM and its derivatives, rank-1 append, greedy append, removal, GP.covar, sampled and batched roll-outs
(ME, TA, EM) with their tangents, leave-one-out cross-validation and its gradient.
    compute-sanitizer --tool racecheck python tools/sanitize_run.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import gp_mpc_b200
from gp_mpc_b200 import _lib as L
from oracle import gp_oracle as orc
from tests._util import relinf

N, Nx, Ny, H = int(os.environ.get('SAN_N', 700)), 5, 2, 21
p = orc.synthetic_problem(N, Nx, Ny, config_id=3, H=H)
eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
eng.set_data(p['X'], p['Y']); eng.set_hyper(p['hyper'])
eng.set_option('small_tiles', 4)          # 128x64 cp.async GEMM for all but the smallest products (TMA: eng_t below)
eng.factorize()
post = orc.postfit(p['X'], p['Y'], p['hyper'], lapack_general_solve=False)
print('chol', relinf(eng.get(L.GET_CHOL, 0), post['chol'][0]), flush=True)
mo, vo = orc.gp_mean_var(p['X'], p['hyper'], post['alpha'], post['chol'], p['Z'])
for ctas in (0, 1, 3, 37):
    eng.set_option('predict_ctas', ctas)
    mean, var, cov, jac = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
    print('predict ctas=%d' % ctas, relinf(mean, mo), relinf(var, vo), flush=True)
eng.set_option('predict_ctas', 0)
ref = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
# gpmpc_predict_device (the entry bench.py times): device inputs and outputs, no host copies, same bits as gpmpc_predict
import torch
dZ, dS = torch.from_numpy(p['Z']).cuda(), torch.from_numpy(p['Sigma']).cuda()
dout = [torch.empty(s, dtype=torch.float64, device='cuda') for s in ((H, Ny), (H, Ny), (H, Ny, Ny), (H, Ny, Nx))]
torch.cuda.synchronize()
eng.predict_device(L.METHOD_TA, H, dZ.data_ptr(), dS.data_ptr(), 0, *[t.data_ptr() for t in dout], sync=True)
print('predict_device', all(np.array_equal(t.cpu().numpy(), r) for t, r in zip(dout, ref)), flush=True)
eng.set_option('predict_ctas', 5)
g = eng.predict_grad(p['Z'], p['Sigma'], L.METHOD_TA, want_hess=True)
fd = orc.predict_grad_fd(p['X'], p['hyper'], post['alpha'], post['chol'], p['Z'], p['Sigma'], 'TA')
print('grad', relinf(g['dvar_dz'], fd['dvar']), relinf(g['dcov_dz'], fd['dcov']), flush=True)
eng.set_option('refine', 1)
mean, var, _, _ = eng.predict(p['Z'], p['Sigma'], L.METHOD_TA)
print('refine', relinf(var, vo), flush=True)
eng.set_option('refine', 0)
m_em, v_em, c_em, _ = eng.predict(p['Z'][:2], 1e-4 * np.eye(Nx), L.METHOD_EM, want_jac=False)
print('em var>0', bool((v_em > 0).all()), flush=True)
eg = eng.predict_em_grad(p['Z'][:2], 1e-4 * np.eye(Nx))
print('em_grad finite', all(bool(np.isfinite(eg[k]).all()) for k in eg), np.array_equal(eg['cov'], c_em), flush=True)
pc = eng.posterior_cov(p['Z'][:5])
sm, _, kept = eng.rollout_sample(p['Z'][:3], np.repeat(p['Z'][:3, None, Ny:], 4, 1), np.ones((3, 4, Ny)))
print('rollout_sample finite', bool(np.isfinite(sm).all()), int(kept.sum()), flush=True)
smg, _, _, dsm = eng.rollout_sample_grad(p['Z'][:3], np.repeat(p['Z'][:3, None, Ny:], 4, 1), np.ones((3, 4, Ny)))
print('rollout_sample_grad finite', bool(np.isfinite(dsm).all()), np.array_equal(smg, sm), flush=True)
# batched roll-outs and their tangents: 'TA' with a feedback gain, 'ME' open loop, and 'EM' one point per chunk
zb, Ub, Sb = p['Z'][:3], np.repeat(p['Z'][:3, None, Ny:], 3, 1), np.tile(1e-4 * np.eye(Nx), (3, 1, 1))
for name, meth, Kb in (('TA K', L.METHOD_TA, 0.1 * np.ones((Nx - Ny, Ny))), ('ME', L.METHOD_ME, None)):
    rb = eng.rollout_batch(zb, Ub, Sb, meth, K=Kb)
    rg = eng.rollout_batch_grad(zb, Ub, Sb, meth, K=Kb)
    print('rollout_batch(_grad) %s' % name, all(np.array_equal(a, b) for a, b in zip(rb, rg)),
          bool(np.isfinite(rg[3]).all() and np.isfinite(rg[4]).all()), flush=True)
eng.set_option('em_points', 1)
re_ = eng.rollout_batch_em(zb[:2], Ub[:2, :2], Sb[:2])
reg = eng.rollout_batch_em_grad(zb[:2], Ub[:2, :2], Sb[:2])
print('rollout_batch_em(_grad)', all(np.array_equal(a, b) for a, b in zip(re_, reg)),
      bool(np.isfinite(reg[3]).all() and np.isfinite(reg[4]).all()), flush=True)
eng.set_option('em_points', 0)
_, _, ln = eng.loo()
fl, gl = eng.loo_nlpp(0, p['hyper'][0] * 0.9, grad=True)
print('loo', ln, fl, bool(np.isfinite(gl).all()), flush=True)
nll, gr = eng.nlml(0, p['hyper'][0] * 0.9, grad=True)
print('nlml', nll, orc.calc_NLL(p['hyper'][0] * 0.9, p['X'], p['Y'][:, 0], False), flush=True)
eng.factorize()
ok = eng.append(p['X'][0] + 0.3, p['Y'][0])
print('append', ok, flush=True)
picked, _, ok = eng.append_greedy(p['Z'][:8], np.zeros((8, Ny)), 3)
eng.remove([0, 5])
print('append_greedy', ok, picked.tolist(), 'remove', eng.N, flush=True)
eng.close()
# the TMA tensor-map GEMM serves products of at least 4 * SMs 128x64 tiles: Npad 1152 with 24 outputs puts the bottom
# panel of the top-level split there (576 tiles)
pt = orc.synthetic_problem(1130, Nx, 24, config_id=4)
eng_t = gp_mpc_b200.Engine(1130, Nx, 24, device=0)
eng_t.set_data(pt['X'], pt['Y']); eng_t.set_hyper(pt['hyper'])
eng_t.factorize()
print('chol (TMA)', relinf(eng_t.get(L.GET_CHOL, 23), orc.factor_large(pt['X'], pt['Y'][:, 23], pt['hyper'][23])['chol']), flush=True)
eng_t.close()
# gpmpc_predict's copy transports: H = 300 points of 16 outputs (Nx = 10) are 1.07 MB of outputs, above the 1 MiB that
# the assembling CTA writes straight into mapped host memory, so the inputs go H2D into dIn and the outputs D2H from dOut
pc_ = orc.synthetic_problem(200, 10, 16, config_id=5)
eng_c = gp_mpc_b200.Engine(200, 10, 16, device=0)
eng_c.set_data(pc_['X'], pc_['Y']); eng_c.set_hyper(pc_['hyper'])
eng_c.factorize()
Zc = 0.5 * np.random.default_rng(5).standard_normal((300, 10))
mc, vc, cc, jc = eng_c.predict(Zc, 1e-4 * np.eye(10), L.METHOD_TA)
_, vj, _, _ = eng_c.predict(Zc, None, L.METHOD_ME, want_cov=False)
print('predict (copy out)', bool(np.isfinite(cc).all()), np.array_equal(vc, vj), flush=True)
eng_c.close()
print('done', flush=True)

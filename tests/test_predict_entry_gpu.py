"""The predict-family entry points share one guard: on a handle that has not been factorised, each one fails with
GPMPC_ERR_STATE and an error that names the entry that was called."""
import numpy as np
import pytest

from tests._util import load_fixture

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('entry', ['predict', 'predict_device', 'posterior_cov', 'predict_grad', 'predict_hess',
                                   'predict_em_grad', 'rollout_batch', 'rollout'])
def test_unfactorised_handle_error_names_the_entry(entry):
    import gp_mpc_b200
    import torch
    L = gp_mpc_b200._lib
    m = load_fixture('tank')
    X, Y, hyper = m['X'], m['Y'], m['hyper']
    (N, Nx), Ny = X.shape, Y.shape[1]
    eng = gp_mpc_b200.Engine(N, Nx, Ny, device=0)
    eng.set_data(X, Y)
    eng.set_hyper(hyper)                          # no factorize
    Z = X[:2] + 0.01
    S = 1e-3 * np.eye(Nx)
    U = np.zeros((2, 3, Nx - Ny))
    dZ, dS = torch.from_numpy(Z).cuda(), torch.from_numpy(S).cuda()
    d_out = [torch.empty(2, Ny, dtype=torch.float64, device='cuda'), torch.empty(2, Ny, dtype=torch.float64, device='cuda'),
             torch.empty(2, Ny, Ny, dtype=torch.float64, device='cuda'), torch.empty(2, Ny, Nx, dtype=torch.float64, device='cuda')]
    torch.cuda.synchronize()
    calls = dict(predict=lambda: eng.predict(Z, S),
                 predict_device=lambda: eng.predict_device(L.METHOD_TA, 2, dZ.data_ptr(), dS.data_ptr(), 0,
                                                           *[t.data_ptr() for t in d_out], sync=True),
                 posterior_cov=lambda: eng.posterior_cov(Z),
                 predict_grad=lambda: eng.predict_grad(Z, S),
                 predict_hess=lambda: eng.predict_hess(Z, S),
                 predict_em_grad=lambda: eng.predict_em_grad(Z, S),
                 rollout_batch=lambda: eng.rollout_batch(Z, U, np.stack([S, S])),
                 rollout=lambda: eng.rollout(Z[0], U[0], S))
    with pytest.raises(L.GpmpcError) as e:
        calls[entry]()
    assert e.value.code == L.ERR_STATE
    assert 'gpmpc_%s: call gpmpc_factorize first' % entry in str(e.value)
    eng.close()

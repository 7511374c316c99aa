"""CPU-side checks: the C-ABI library loads and exports every symbol include/gpmpc.h
declares, refuses to run without a GPU (no CPU fallback), and the host-side partition /
driver logic is right."""
import ctypes
import os
import re

import numpy as np
import pytest
from tests._engines import built_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    L = built_lib()
    lib = L.load()
    hdr = open(os.path.join(ROOT, 'include', 'gpmpc.h')).read()
    declared = set(re.findall(r'\b(gpmpc_[A-Za-z_0-9]+)\s*\(', hdr))
    # the CasADi `external` family (function + Jacobian function) of include/gpmpc_casadi.h
    hdr2 = open(os.path.join(ROOT, 'include', 'gpmpc_casadi.h')).read().split('#ifndef GPMPC_CASADI_H')[1]
    declared |= set(re.findall(r'\b((?:jac_)?gp_b200[A-Za-z_0-9]*)\s*\(', hdr2))
    assert {'gp_b200', 'jac_gp_b200', 'gp_b200_bind', 'gp_b200_sparsity_out', 'jac_gp_b200_work'} <= declared
    bound = {s[0] for s in L.SYMBOLS}
    assert declared == bound, (declared ^ bound)
    for name in declared:
        assert getattr(lib, name) is not None
    assert lib.gpmpc_version() >= 100


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    L = built_lib()
    with pytest.raises(L.GpmpcError) as e:
        L.Engine(10, 2, 1)
    assert 'no CPU path' in str(e.value)
    h = ctypes.c_void_p()
    assert L.load().gpmpc_create(0, 2, 1, 0, 1, 0, ctypes.byref(h)) == L.ERR_ARG
    # product package never imports the oracle
    for root, _, files in os.walk(os.path.join(ROOT, 'gp-mpc_b200')):
        for f in files:
            if f.endswith(('.py', '.cu', '.cuh')):
                assert 'oracle' not in open(os.path.join(root, f)).read().replace('oracle = ', ''), f


def test_partition_index_work():
    from gp_mpc_b200.partition import choose_mode, output_block, point_block
    for Ny in range(1, 20):
        for W in (1, 2, 3, 4, 8):
            blocks = [output_block(Ny, r, W) for r in range(W)]
            owned = [a for b, n in blocks for a in range(b, b + n)]
            assert owned == list(range(Ny))                      # exact cover, in order
            per = -(-Ny // W)
            assert all(b == min(Ny, r * per) for r, (b, n) in enumerate(blocks))
            mode = choose_mode(Ny, W)
            assert mode == ('outputs' if all(n > 0 for _, n in blocks) else 'points')
    assert choose_mode(8, 8) == 'outputs' and choose_mode(6, 8) == 'points' and choose_mode(6, 4) == 'points'
    assert choose_mode(6, 2) == 'outputs' and choose_mode(6, 3) == 'outputs'
    for H in (1, 7, 30, 50):
        for W in (1, 2, 4, 8):
            pts = [i for r in range(W) for i in range(point_block(H, r, W)[0], sum(point_block(H, r, W)))]
            assert pts == list(range(H))


def test_bounds_and_init_follow_the_reference():
    from gp_mpc_b200.optimize import bounds_and_init, count_mean_params
    from oracle import gp_oracle as orc
    rng = np.random.default_rng(0)
    X = rng.standard_normal((30, 4)); y = rng.standard_normal(30)
    b, i = bounds_and_init(X, y)
    bo, io = orc.train_bounds_init(X, y)
    assert np.array_equal(b, bo) and np.array_equal(i, io)
    assert b[0, 0] == -1.0                                         # the reference's `1-2` typo (q7)
    assert bounds_and_init(X, y, fixed_bounds=True)[0][0, 0] == 1e-2
    assert [count_mean_params(m, 4) for m in ('zero', 'const', 'linear', 'polynomial')] == [0, 1, 5, 9]
    with pytest.raises(NameError):
        count_mean_params('cubic', 4)


def test_bench_workload_generator_matches_the_oracle_generator():
    import bench
    from oracle import gp_oracle as orc
    a = bench.make_workload(50, 4, 2, 3, 7)
    b = orc.synthetic_problem(50, 4, 2, config_id=3, H=7)
    for k in ('X', 'Y', 'hyper', 'Z', 'Sigma'):
        assert np.array_equal(a[k], b[k])
    assert set(bench.WORKLOADS) == {'c2', 'c3', 'c5'}


def test_casadi_external_metadata_without_a_gpu():
    """The `casadi.external` helper functions answer without a device; patterns exist only once bound."""
    lib = built_lib().load()
    assert lib.gp_b200_n_in() == 2 and lib.gp_b200_n_out() == 2
    assert lib.jac_gp_b200_n_in() == 4 and lib.jac_gp_b200_n_out() == 4
    assert [lib.gp_b200_name_in(i) for i in range(2)] == [b'z', b'sigma']
    assert [lib.jac_gp_b200_name_out(i) for i in range(4)] == [b'jac_mean_z', b'jac_mean_sigma', b'jac_cov_z', b'jac_cov_sigma']
    assert not lib.gp_b200_sparsity_in(0) and not lib.jac_gp_b200_sparsity_out(2)      # not bound
    sz = [ctypes.c_longlong(-1) for _ in range(4)]
    assert lib.gp_b200_work(*[ctypes.byref(x) for x in sz]) == 0 and [x.value for x in sz] == [2, 2, 0, 0]
    assert lib.gp_b200_bind(None, 1, 5) != 0
